#!/usr/bin/env python
"""bench.py — decode tokens/sec (+ p50 TTFT) of the TGIS hot path on H100.

A "step" = one pass of the hot path over one batch of synthetic input = one whole batched generation job:
B concurrent requests x (512-token prompt -> 128 generated tokens), greedy, on synthetic seeded weights of the named
architecture (BASELINE.json configs[1]: Llama-3-8B bf16, 1xH100, batch 32, 512-in/128-out).

  value  : decode tokens/s with inputs resident in HBM — tokens sampled in pure-decode engine steps divided by the
           CUDA-event time of those steps (events on the engine's launching stream), max over ranks.
  e2e    : the same metric through the public C-ABI call with HOST buffers (tgis_engine_add_request /
           run_until_idle / poll): wall clock of the decode phase, i.e. including the per-step H2D metadata copy, the
           D2H result copy and the host scheduler.  Also reports whole-job output tokens/s and p50 TTFT.
  roofline: dominant kernel = the wgmma GEMM; achieved = algorithmic bytes / CUDA-event time per launch, measured in
           a separate short profiled pass (events around every GEMM launch), against the H100 SXM data-sheet HBM3
           bandwidth (3.35 TB/s);
           decode_step_frac_of_hbm_roofline = algorithmic bytes of one decode step / measured step time / peak.
  cpu_baseline / --impl reference: the CPU oracle (oracle/llama_oracle.py — the port of the reference's vLLM-CPU path,
           which cannot be built offline; BASELINE.md §4) timed on the host cores on a bounded sample.

N > 1 (torchrun): ONE tensor-parallel engine over the N GPUs (north_star's shape: column-parallel qkv / gate_up,
row-parallel o / down with the fused push all-reduce + residual + RMSNorm exchange kernel, vocab-parallel lm_head) on
the SAME workload as N = 1 -> "scaling": "strong"; `tp_parity` compares its greedy tokens with a single-GPU engine in
the same run.  Secondary fields: `dp` (independent replicas, weak scaling: the faster way to use N GPUs for a model that
fits one), `named_configs` (N = 4: BASELINE configs[3]; N = 8: configs[4], Llama-3-70B TP = 8, 256 requests),
--parallel dp restores the replicas-only run.

--dump-outputs DIR: after the timed steps, the token ids the last timed step generated ([batch, gen_len] float64, rows in
request order; rank 0's requests when N > 1) are written to DIR/tokens.npy.  They are the timed path's whole output: its
requests ask for no logprobs (num_logprobs = 0), so the engine computes none.  Weights, prompts and
sampling are seeded, so two builds given the same arguments can be compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--model", default="llama3-8b")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--prompt-len", type=int, default=512)
    ap.add_argument("--gen-len", type=int, default=128)
    ap.add_argument("--parallel", default=None, choices=["dp", "tp"],
                    help="N>1: tp (default) = ONE tensor-parallel engine over the N GPUs, strong scaling of the N=1 "
                         "workload (north_star's TP shape; the dp number is reported as a secondary field); "
                         "dp = independent replicas only (weak scaling)")
    ap.add_argument("--named-configs", default="auto", choices=["auto", "none", "force", "0", "1"],
                    help="auto: N=4 also runs BASELINE.json configs[3] (8B TP=4, 128 requests, mixed lengths), N=8 also "
                         "configs[4] (70B TP=8, 256 requests), reported under named_configs; force: both legs at any N>1 "
                         "(with --layers: a cheap check of the code paths); none: skip")
    ap.add_argument("--max-batched-tokens", type=int, default=2048,
                    help="scheduler token budget per step (= chunked-prefill size); 2048 = this engine's and vLLM's "
                         "online-serving default")
    ap.add_argument("--sampling", default="greedy", choices=["greedy", "cfg3"],
                    help="cfg3 = repetition penalty 1.2 + length penalty (64, 1.05) + typical_p 0.9 sampling")
    ap.add_argument("--layers", type=int, default=0, help="experiments: override the preset's layer count")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--cpu-layers", type=int, default=8, help="layers timed by the CPU baseline (extrapolated)")
    ap.add_argument("--cpu-steps", type=int, default=20, help="decode steps of the ours-arm cpu_baseline leg")
    ap.add_argument("--cpu-budget-s", type=float, default=60.0, help="wall-clock bound of the CPU baseline sample")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the last timed step's generated token ids to DIR/tokens.npy (rank 0)")
    return ap.parse_args()


_T0 = time.time()


def log(msg: str) -> None:
    print(f"[bench +{time.time() - _T0:7.1f}s] {msg}", file=sys.stderr, flush=True)


def peaks() -> tuple[float, str]:
    return 3350.0, "NVIDIA H100 SXM data sheet (HBM3, 700 W part); not measured"


class ClockSampler:
    """nvidia-smi clocks + throttle reasons during the timed region."""

    def __init__(self, index: int):
        self.index = index
        self.samples: list[tuple[float, float, str]] = []
        self._stop = threading.Event()
        self._t: threading.Thread | None = None

    def _run(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                                      str(self.index)], capture_output=True, text=True, timeout=5).stdout.strip()
                f = [x.strip() for x in out.split(",")]
                reasons = [n for n, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                                              "sw_power_cap"), f[2:6]) if v.lower().startswith("active")]
                self.samples.append((float(f[0]), float(f[1]), ",".join(reasons)))
            except Exception:  # noqa: BLE001
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        if self._t:
            self._t.join(timeout=6)

    def summary(self) -> dict:
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        reasons = sorted({r for s in self.samples for r in s[2].split(",") if r})
        return {"sm_mhz": statistics.median(s[0] for s in self.samples), "sm_max_mhz": self.samples[0][1],
                "reasons": reasons, "samples": len(self.samples)}


# ----------------------------------------------------------------------------------------------------- CPU reference
def cpu_reference(args, steps: int, warmup: int, budget_s: float | None = None) -> dict:
    """The oracle port of the reference's CPU path on the host cores, bounded sample.  One "step" = ONE batched decode
    step of B sequences with a prompt_len-token (synthetic) KV history through `cpu_layers` of the model's layers +
    final norm + lm_head + greedy sampling (log-softmax + argmax, the oracle's sampler path); the per-layer time is
    extrapolated linearly to the full depth (stated in `sample`).  Thread count is fixed (min(cores, 32): wider is
    slower on the pool's 128-thread hosts because of OpenMP fork/join), the statistic is the MEDIAN step time, and one
    512-token prefill is timed for a TTFT estimate -- so the ours-arm `cpu_baseline` and the `--impl reference` arm
    measure the same thing the same way."""
    import dataclasses

    import torch

    if args.model.startswith("opt-"):
        return cpu_reference_opt(args, steps, warmup, budget_s)
    from oracle.llama_oracle import CONFIGS, LlamaOracle, SeqState

    cfg_full = CONFIGS[args.model]
    L_s = min(cfg_full.n_layers, args.cpu_layers)
    cfg = dataclasses.replace(cfg_full, n_layers=L_s)
    cores = os.cpu_count() or 1
    threads = int(os.environ.get("TGIS_CPU_THREADS", min(cores, 32)))
    torch.set_num_threads(threads)
    g = torch.Generator().manual_seed(0)
    # vLLM's CPU backend runs bf16 where the host has AMX / avx512_bf16 and fp32 otherwise: pick by a micro-benchmark
    xa, wa = torch.randn(32, 4096), torch.randn(4096, 4096)

    def _t(dt):
        x_, w_ = xa.to(dt), wa.to(dt)
        for _ in range(2):
            torch.nn.functional.linear(x_, w_)
        t0 = time.perf_counter()
        for _ in range(5):
            torch.nn.functional.linear(x_, w_)
        return time.perf_counter() - t0

    t16, t32 = _t(torch.bfloat16), _t(torch.float32)
    dtype = torch.bfloat16 if t16 <= 1.5 * t32 else torch.float32
    log(f"cpu reference: linear micro-bench bf16 {1e3 * t16:.1f} ms vs fp32 {1e3 * t32:.1f} ms -> {dtype}, {threads} threads")
    tile = (torch.randn(1024, 1024, generator=g) * 0.02).to(dtype)

    def fake(rows: int, cols: int) -> torch.Tensor:  # values irrelevant for timing; avoids minutes of randn
        r = (rows + 1023) // 1024
        c = (cols + 1023) // 1024
        return tile.repeat(r, c)[:rows, :cols].contiguous()

    w = {"model.embed_tokens.weight": fake(cfg.vocab, cfg.hidden), "lm_head.weight": fake(cfg.vocab, cfg.hidden),
         "model.norm.weight": torch.ones(cfg.hidden, dtype=dtype)}
    for i in range(cfg.n_layers):
        p = f"model.layers.{i}."
        w[p + "self_attn.q_proj.weight"] = fake(cfg.q_dim, cfg.hidden)
        w[p + "self_attn.k_proj.weight"] = fake(cfg.kv_dim, cfg.hidden)
        w[p + "self_attn.v_proj.weight"] = fake(cfg.kv_dim, cfg.hidden)
        w[p + "self_attn.o_proj.weight"] = fake(cfg.hidden, cfg.q_dim)
        w[p + "mlp.gate_proj.weight"] = fake(cfg.ffn, cfg.hidden)
        w[p + "mlp.up_proj.weight"] = fake(cfg.ffn, cfg.hidden)
        w[p + "mlp.down_proj.weight"] = fake(cfg.hidden, cfg.ffn)
        w[p + "input_layernorm.weight"] = torch.ones(cfg.hidden, dtype=dtype)
        w[p + "post_attention_layernorm.weight"] = torch.ones(cfg.hidden, dtype=dtype)
    ora = LlamaOracle(cfg, w, dtype=dtype)
    del w
    B, ctx = args.batch, args.prompt_len
    sts = []
    for _ in range(B):
        st = SeqState(cfg, dtype)
        st.k = [fake(ctx, cfg.kv_dim).view(ctx, cfg.n_kv_heads, cfg.head_dim) for _ in range(cfg.n_layers)]
        st.v = [fake(ctx, cfg.kv_dim).view(ctx, cfg.n_kv_heads, cfg.head_dim) for _ in range(cfg.n_layers)]
        st.n = ctx
        sts.append(st)
    toks = [5] * B

    def one_step():
        nonlocal toks
        t0 = time.perf_counter()
        logits = ora.step([(st, [t]) for st, t in zip(sts, toks)])
        lp = torch.log_softmax(logits, dim=-1)                 # raw logprobs (S1) + greedy argmax (S4)
        toks = torch.argmax(lp, dim=-1).tolist()
        return time.perf_counter() - t0

    times = []
    t_end = time.perf_counter() + (budget_s if budget_s else 1e9)
    for it in range(warmup + steps):
        t = one_step()
        if it >= warmup:
            times.append(t)
        if time.perf_counter() > t_end and len(times) >= 3:
            break
    t_step = statistics.median(times)
    log(f"cpu reference: {len(times)} timed {L_s}-layer decode steps, median {t_step:.3f} s "
        f"(min {min(times):.3f}, max {max(times):.3f})")
    # head (final norm + lm_head + sampling) timed alone so the layer part can be scaled to the full depth
    xh = torch.randn(B, cfg.hidden).to(dtype)

    def head_once():
        t0 = time.perf_counter()
        torch.argmax(torch.log_softmax(ora.head(xh), dim=-1), dim=-1)
        return time.perf_counter() - t0

    head_once()
    t_head = statistics.median(head_once() for _ in range(5))
    t_layer = max(t_step - t_head, 0.0) / L_s
    t_full = t_head + t_layer * cfg_full.n_layers
    # TTFT estimate: one 512-token prompt through the timed layers, scaled to the full depth; a burst of B prompts served
    # FIFO one prompt at a time has p50 TTFT ~ (B + 1) / 2 prompts
    t0 = time.perf_counter()
    ora.step([(ora.new_seq(), [7] * ctx)])
    t_pf = (time.perf_counter() - t0 - t_head) / L_s * cfg_full.n_layers + t_head
    val = B / t_full
    return {"value": val, "unit": "tokens/s", "cores": threads, "kind": "port",
            "sample": f"{args.model} B={B} ctx={ctx} (synthetic KV history): {L_s} of {cfg_full.n_layers} layers + lm_head + "
                      f"greedy sampling timed over {len(times)} batched decode steps (median {t_step * 1e3:.0f} ms/step, head "
                      f"{t_head * 1e3:.0f} ms), per-layer time extrapolated linearly to {cfg_full.n_layers} layers; one "
                      f"{ctx}-token prefill timed the same way; torch CPU {str(dtype).split('.')[-1]} oracle "
                      f"(oracle/llama_oracle.py), {threads} of {cores} threads",
            "ms_per_step": 1e3 * t_full, "sample_ms_per_step": 1e3 * t_step, "prefill_one_prompt_s": t_pf, "ttft_p50_est_ms": 1e3 * t_pf * (B + 1) / 2,
            "step_times_s": [round(t, 4) for t in times]}


def cpu_reference_opt(args, steps: int, warmup: int, budget_s: float | None = None) -> dict:
    """BASELINE configs[0] on the architecture it names (facebook/opt-125m dims, seeded random weights): the OPT oracle
    (oracle/opt_oracle.py) timed IN FULL on the host cores -- all layers, the real prefill of every prompt, then real
    batched decode steps with greedy sampling until gen_len tokens or the time budget; no extrapolation."""
    import numpy as np
    import torch

    from oracle.opt_oracle import OPT_CONFIGS, OPTOracle, synthetic_opt_weights

    cfg = OPT_CONFIGS[args.model]
    cores = os.cpu_count() or 1
    threads = int(os.environ.get("TGIS_CPU_THREADS", min(cores, 32)))
    torch.set_num_threads(threads)
    ora = OPTOracle(cfg, synthetic_opt_weights(cfg, seed=7))
    B, P, G = args.batch, args.prompt_len, args.gen_len
    rng = np.random.RandomState(1234)
    prompts = [rng.randint(3, cfg.vocab, size=P).tolist() for _ in range(B)]
    sts = [ora.new_seq() for _ in range(B)]
    t0 = time.perf_counter()
    toks, ttfts = [], []
    for st, p in zip(sts, prompts):   # prompts served FIFO, one prefill each (the reference engine's CPU scheduler)
        toks.append(int(torch.argmax(torch.log_softmax(ora.step([(st, p)])[0], -1))))
        ttfts.append(time.perf_counter() - t0)
    times = []
    t_end = time.perf_counter() + (budget_s if budget_s else 1e9)
    for it in range(G - 1):
        t1 = time.perf_counter()
        logits = ora.step([(st, [t]) for st, t in zip(sts, toks)])
        toks = torch.argmax(torch.log_softmax(logits, -1), -1).tolist()
        times.append(time.perf_counter() - t1)
        if time.perf_counter() > t_end and len(times) >= max(3, steps):
            break
    t_step = statistics.median(times)
    return {"value": B / t_step, "unit": "tokens/s", "cores": threads, "kind": "port",
            "sample": f"{args.model} (all {cfg.n_layers} layers) B={B}: {P}-token prefill of every prompt + {len(times)} real "
                      f"batched decode steps with greedy sampling, nothing extrapolated; torch CPU bfloat16 oracle "
                      f"(oracle/opt_oracle.py), {threads} of {cores} threads",
            "ms_per_step": 1e3 * t_step, "sample_ms_per_step": 1e3 * t_step, "prefill_one_prompt_s": ttfts[0],
            "ttft_p50_est_ms": 1e3 * statistics.median(ttfts), "step_times_s": [round(t, 4) for t in times[:64]]}


def reduce_over_ranks(max_vals: list[float], sum_vals: list[float], device: str) -> tuple[list[float], list[float]]:
    """Whole-job aggregation for the N>1 (data-parallel replicas) path: times -> MAX over ranks, counts -> SUM.
    Works on any initialised torch.distributed backend (NCCL on the GPU box, gloo in tests/test_multirank_cpu.py)."""
    import torch
    import torch.distributed as dist

    vals = torch.tensor(max_vals, dtype=torch.float64, device=device)
    sums = torch.tensor(sum_vals, dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(vals, op=dist.ReduceOp.MAX)
        dist.all_reduce(sums, op=dist.ReduceOp.SUM)
    return vals.tolist(), sums.tolist()


# ----------------------------------------------------------------------------------------------------------- ours
METRIC = "decode tokens/sec + p50 TTFT, 512-in/128-out batch, 1/2/4/8xH100 vs CPU ref"


def _load_synthetic(eng, cfg, seed: int) -> None:
    """Seeded N(0, 0.02) weights generated on the device, one tensor at a time ("PyTorch tensors for weights only").
    Under tensor parallelism every rank draws the SAME full tensor (same seed) and the engine keeps its shard."""
    import torch

    if getattr(cfg, "arch", "llama") == "opt":   # --model opt-125m (BASELINE configs[0] on the architecture it names)
        from vllm_tgis_adapter_b200.engine.loader import load_synthetic_weights

        load_synthetic_weights(eng, cfg, seed, torch.cuda.current_device())
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return
    gen = torch.Generator(device="cuda").manual_seed(seed)

    def rnd(r, c):
        return (torch.randn(r, c, generator=gen, device="cuda", dtype=torch.float32) * 0.02).to(torch.bfloat16)

    q_dim, kv_dim = cfg.n_q_heads * 128, cfg.n_kv_heads * 128
    ones = torch.ones(cfg.hidden, dtype=torch.bfloat16, device="cuda")
    eng.load_weight("model.embed_tokens.weight", rnd(cfg.vocab, cfg.hidden))
    eng.load_weight("lm_head.weight", rnd(cfg.vocab, cfg.hidden))
    eng.load_weight("model.norm.weight", ones)
    for i in range(cfg.n_layers):
        p = f"model.layers.{i}."
        eng.load_weight(p + "self_attn.q_proj.weight", rnd(q_dim, cfg.hidden))
        eng.load_weight(p + "self_attn.k_proj.weight", rnd(kv_dim, cfg.hidden))
        eng.load_weight(p + "self_attn.v_proj.weight", rnd(kv_dim, cfg.hidden))
        eng.load_weight(p + "self_attn.o_proj.weight", rnd(cfg.hidden, q_dim))
        eng.load_weight(p + "mlp.gate_proj.weight", rnd(cfg.ffn, cfg.hidden))
        eng.load_weight(p + "mlp.up_proj.weight", rnd(cfg.ffn, cfg.hidden))
        eng.load_weight(p + "mlp.down_proj.weight", rnd(cfg.hidden, cfg.ffn))
        eng.load_weight(p + "input_layernorm.weight", ones)
        eng.load_weight(p + "post_attention_layernorm.weight", ones)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


_ENGINE_SEQ = [0]


def _build_engine(model: str, *, max_seqs: int, max_len: int, kv_tokens: int, max_batched: int, tp: int, rank: int,
                  local: int, weight_seed: int, layers: int = 0):
    """One engine (tp == 1) or this rank's shard of ONE tensor-parallel engine over `tp` GPUs."""
    import dataclasses

    import torch

    from vllm_tgis_adapter_b200.engine.core import PRESETS, NativeEngine

    cfg = dataclasses.replace(PRESETS[model], max_model_len=max_len)
    if layers > 0:
        cfg = dataclasses.replace(cfg, n_layers=layers)
    blocks = max(kv_tokens, max_len + 64) // 32 + 2 * max_seqs   # at least one max_model_len sequence (batch-1 runs)
    kv_bytes = int(blocks * 2 * cfg.n_layers * (cfg.n_kv_heads // tp) * 32 * 128 * 2 * 1.1)
    tp_kw = {}
    if tp > 1:
        import torch.distributed as dist

        _ENGINE_SEQ[0] += 1
        ids = [NativeEngine.nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0, device=torch.device("cuda", local))
        tp_kw = dict(tp_size=tp, tp_rank=rank, nccl_id=ids[0],
                     shm_name=f"/tgis_bench_{os.environ.get('MASTER_PORT', '0')}_{_ENGINE_SEQ[0]}")
    eng = NativeEngine(cfg, max_num_seqs=max_seqs, max_batched_tokens=max_batched, kv_cache_bytes=kv_bytes, device=local,
                       seed=1234, **tp_kw)
    _load_synthetic(eng, cfg, weight_seed)
    return eng, cfg


def _sampling(kind: str, G: int):
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    if kind == "cfg3":   # BASELINE.json configs[2]: repetition penalty + ExpDecayLengthPenalty + typical-p sampling
        return make_sampling_params(greedy=False, temperature=1.0, typical_p=0.9, repetition_penalty=1.2,
                                    length_penalty=(64, 1.05), seed=1234, max_tokens=G, min_tokens=G, eos_token_id=2)
    return make_sampling_params(greedy=True, max_tokens=G, min_tokens=G, eos_token_id=2)


def _job(eng, prompts, sp):
    """One bench step through the C ABI with host buffers.  Returns (decode_wall_s, ttfts, n_tokens, n_tokens produced
    inside the decode wall, per-request token ids): the decode phase starts when the LAST request has its first token;
    tokens that early requests produced before that (chunked prefill interleaves them) are not counted in it."""
    for i, pr in enumerate(prompts):
        eng.add_request(f"r{i}", pr, sp)
    eng.run_until_idle()
    t_end = time.monotonic()
    first, n_tok, stamps = {}, 0, []
    toks: list[list[int]] = [[] for _ in prompts]
    while True:
        outs = eng.poll(0)
        if not outs:
            break
        for o in outs:
            if o.new_token is not None:
                n_tok += 1
                stamps.append(o.ts_last_token)
                toks[int(o.request_id[1:])].append(o.new_token)
            first[o.request_id] = (o.ts_first_token, o.ts_arrival)
    t_all_first = max(v[0] for v in first.values())
    ttfts = [v[0] - v[1] for v in first.values()]
    return t_end - t_all_first, ttfts, n_tok, sum(1 for t in stamps if t > t_all_first), toks


def _timed_jobs(eng, prompts, sp, warmup: int, steps: int, barrier, clock_index: int | None, tag: str) -> dict:
    for i in range(warmup):
        dw, tt, nt, _, _ = _job(eng, prompts, sp)
        log(f"{tag} warmup job {i}: {nt} tokens, decode wall {dw:.3f}s, ttft p50 {1e3 * statistics.median(tt):.1f} ms")
    barrier()
    st0 = eng.status()
    decode_wall, ttfts, n_tok, n_tok_dec, toks = 0.0, [], 0, 0, None
    sampler = ClockSampler(clock_index) if clock_index is not None else None
    if sampler:
        sampler.__enter__()
    t0 = time.perf_counter()
    for _ in range(steps):
        dw, tt, nt, nd, toks = _job(eng, prompts, sp)
        decode_wall += dw
        ttfts += tt
        n_tok += nt
        n_tok_dec += nd
    barrier()
    wall = time.perf_counter() - t0
    if sampler:
        sampler.__exit__()
    st1 = eng.status()
    return {"dec_ms": st1.gpu_decode_ms - st0.gpu_decode_ms, "dec_tok": st1.decode_tokens - st0.decode_tokens,
            "dec_steps": st1.decode_steps - st0.decode_steps, "launches": st1.kernel_launches - st0.kernel_launches,
            "h2d": (st1.h2d_bytes - st0.h2d_bytes) / steps, "d2h": (st1.d2h_bytes - st0.d2h_bytes) / steps,
            "graph_launches": st1.graph_launches - st0.graph_launches, "steps_total": st1.steps - st0.steps,
            "wall": wall, "decode_wall": decode_wall, "ttfts": ttfts, "n_tok": n_tok, "n_tok_dec": n_tok_dec,
            "tokens": toks, "clocks": sampler.summary() if sampler else None}


def _profiled_pass(eng, prompts, G_short: int = 17) -> dict:
    """Roofline leg: a short pass with CUDA events around every GEMM launch (and every tensor-parallel exchange) of
    the pure-decode steps."""
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    eng.set_profiling(2)
    sp_short = make_sampling_params(greedy=True, max_tokens=G_short, min_tokens=G_short, eos_token_id=2)
    g0 = eng.status()
    for i, pr in enumerate(prompts):
        eng.add_request(f"p{i}", pr, sp_short)
    eng.run_until_idle()
    while eng.poll(0):
        pass
    g1 = eng.status()
    eng.set_profiling(False)
    return {"gemm_ms": g1.gemm_ms - g0.gemm_ms, "gemm_bytes": g1.gemm_bytes - g0.gemm_bytes,
            "gemm_calls": g1.gemm_calls - g0.gemm_calls, "exchange_ms": g1.exchange_ms - g0.exchange_ms,
            "exchange_calls": g1.exchange_calls - g0.exchange_calls,
            "decode_steps": g1.decode_steps - g0.decode_steps,
            "decode_ms": g1.gpu_decode_ms - g0.gpu_decode_ms}


def _teacher_forced_parity(eng, prompts, tokens) -> dict:
    """Score `tokens[i]` (another engine's greedy continuation of prompts[i]) with `eng`: one request per sequence with
    prompt = prompt + tokens and prompt_logprobs = 1; for every generated position the record holds the token's logprob
    and eng's own top-1 at that position."""
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    sp = make_sampling_params(greedy=True, max_tokens=1, num_logprobs=1, prompt_logprobs=1, eos_token_id=2)
    for i, (p, t) in enumerate(zip(prompts, tokens)):
        eng.add_request(f"t{i}", p + t, sp)
    eng.run_until_idle()
    n, top1, worst, gaps = 0, 0, 0.0, []
    while True:
        outs = eng.poll(0)
        if not outs:
            break
        for o in outs:
            i = int(o.request_id[1:])
            if o.prompt_pos >= len(prompts[i]):
                n += 1
                if o.topn and o.topn[0][0] == o.token_id:
                    top1 += 1
                elif o.topn:
                    gaps.append(o.topn[0][1] - o.logprob)
    return {"tokens_scored": n, "is_single_gpu_argmax": top1, "not_argmax": len(gaps),
            "max_logprob_gap_to_argmax": max(gaps) if gaps else 0.0,
            "mean_logprob_gap_to_argmax": (sum(gaps) / len(gaps)) if gaps else 0.0}


def _step_bytes(cfg, B: int, mean_ctx: float, tp: int) -> float:
    """Algorithmic bytes of one decode step PER GPU (SURVEY.md section 8d): weights/tp + KV/tp + one bf16 logits scan."""
    if getattr(cfg, "arch", "llama") == "opt":
        # algorithmic = the model's own dims (64-dim heads); the engine streams zero-padded 128-dim head slots, which shows
        # up as a lower roofline fraction, not as smaller algorithmic bytes
        n_params = cfg.n_layers * (4 * cfg.hidden * cfg.hidden + 2 * cfg.hidden * cfg.ffn) + cfg.vocab * cfg.hidden
        kv_tok = 2 * cfg.n_layers * cfg.n_kv_heads * cfg.head_dim * 2
        return (n_params * 2 + B * mean_ctx * kv_tok) / tp + B * cfg.vocab * 2
    q_dim, kv_dim = cfg.n_q_heads * 128, cfg.n_kv_heads * 128
    n_params = cfg.n_layers * (cfg.hidden * (q_dim + 2 * kv_dim) + cfg.hidden * q_dim + 3 * cfg.hidden * cfg.ffn) \
        + cfg.vocab * cfg.hidden
    kv_tok = 2 * cfg.n_layers * cfg.n_kv_heads * 128 * 2
    return (n_params * 2 + B * mean_ctx * kv_tok) / tp + B * cfg.vocab * 2


def _dump_outputs(out_dir: str, leg: dict) -> None:
    """What a caller of the timed path received in its last step: every request's generated token ids."""
    import numpy as np

    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    np.save(d / "tokens.npy", np.array(leg["tokens"], dtype=np.float64))


def run_ours(args) -> dict | None:
    import numpy as np
    import torch

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    B, P, G = args.batch, args.prompt_len, args.gen_len
    parallel = args.parallel or ("tp" if world > 1 else "dp")
    tp = world if (parallel == "tp" and world > 1) else 1
    max_len = max(1024, P + G + 64)

    def barrier_dp():
        torch.cuda.synchronize()
        if world > 1 and tp == 1:
            dist.barrier()

    def barrier_local():
        torch.cuda.synchronize()

    def prompts_for(cfg, n, seed, lo=None, hi=None):
        rs = np.random.RandomState(seed)
        if lo is None:
            return [rs.randint(1000, cfg.vocab - 1000, size=P).tolist() for _ in range(n)]
        lens = rs.randint(lo, hi + 1, size=n)
        return [rs.randint(1000, cfg.vocab - 1000, size=int(L)).tolist() for L in lens]

    # ============================================================ primary leg: BASELINE configs[1] on N GPUs
    nc = {"0": "none", "1": "auto"}.get(args.named_configs, args.named_configs)
    do_cfg3 = tp > 1 and args.model == "llama3-8b" and (nc == "force" or (nc == "auto" and tp == 4))
    do_cfg4 = tp > 1 and (nc == "force" or (nc == "auto" and world == 8))
    named_b = 128 if do_cfg3 else 0   # configs[3] shares the primary engine
    eng, cfg = _build_engine(args.model, max_seqs=max(B, named_b), max_len=max_len,
                             kv_tokens=max(B, named_b) * (P + G + 32), max_batched=args.max_batched_tokens, tp=tp,
                             rank=rank, local=local, weight_seed=1234 + (rank if tp == 1 else 0), layers=args.layers)
    log(f"engine built and {cfg.n_layers}-layer synthetic weights loaded (tp={tp})")
    primary = prof = named = None
    if tp > 1 and rank != 0:   # tensor-parallel worker: follow rank 0's step plans until it closes its engine
        eng.worker_run()
        eng.close()
    else:
        prompts = prompts_for(cfg, B, 1234 + (rank if tp == 1 else 0))
        sp = _sampling(args.sampling, G)
        primary = _timed_jobs(eng, prompts, sp, args.warmup, args.steps, barrier_dp if tp == 1 else barrier_local, local,
                              "primary")
        log(f"timed region done: {args.steps} jobs in {primary['wall']:.3f}s")
        if args.dump_outputs and rank == 0:
            _dump_outputs(args.dump_outputs, primary)
        prof = _profiled_pass(eng, prompts)
        log(f"profiled pass done: {prof['gemm_calls']} GEMM launches, {prof['gemm_ms']:.2f} ms")
        if named_b:   # BASELINE configs[3]: 8B TP=4, 128 concurrent requests, mixed prompt lengths, continuous batching
            pm = prompts_for(cfg, named_b, 4321, 64, 512)
            r = _timed_jobs(eng, pm, _sampling("greedy", G), 1, 2, barrier_local, None, "cfg[3]")
            pr = _profiled_pass(eng, pm)
            mean_ctx = float(np.mean([len(x) for x in pm])) + G / 2
            by = _step_bytes(cfg, named_b, mean_ctx, tp)
            sm = r["dec_ms"] / max(r["dec_steps"], 1)
            named = {"config": f"BASELINE.json configs[3]: llama3-8b bf16 TP={tp}, 128 concurrent requests submitted together, "
                               "prompt lengths uniform in [64, 512] (seed 4321), 128 new tokens each, greedy, continuous "
                               "batching with chunked prefill",
                     "decode_tokens_per_s": r["dec_tok"] / (r["dec_ms"] * 1e-3),
                     "job_output_tokens_per_s": r["n_tok"] / r["wall"], "decode_step_ms": sm,
                     "ttft_p50_ms": 1e3 * statistics.median(r["ttfts"]),
                     "decode_step_algorithmic_bytes_per_gpu": by,
                     "decode_step_frac_of_hbm_roofline": by / (sm * 1e-3) / 1e9 / peaks()[0] if sm else None,
                     "exchange_ms_per_step": pr["exchange_ms"] / max(pr["decode_steps"], 1),
                     "exchanges_per_step": pr["exchange_calls"] / max(pr["decode_steps"], 1),
                     "gemm_ms_per_step": pr["gemm_ms"] / max(pr["decode_steps"], 1), "jobs_timed": 2}
            log(f"cfg[3] leg done: {named['decode_tokens_per_s']:.0f} tok/s")
        eng.close()
    if world > 1:
        dist.barrier()

    # ============================================================ N > 1: secondary legs
    dp_leg = parity = named70 = None
    if tp > 1:
        # (a) data-parallel replicas of the same workload (weak scaling; what round 1 reported) + the N=1 tokens for the
        #     in-run parity check of the tensor-parallel engine
        e1, c1 = _build_engine(args.model, max_seqs=B, max_len=max_len, kv_tokens=B * (P + G + 32),
                               max_batched=args.max_batched_tokens, tp=1, rank=rank, local=local, weight_seed=1234,
                               layers=args.layers)
        pr1 = prompts_for(c1, B, 1234)     # every replica runs rank 0's prompt set: rank 0's tokens are the N=1 reference

        def barrier_all():
            torch.cuda.synchronize()
            dist.barrier()

        r1 = _timed_jobs(e1, pr1, _sampling(args.sampling, G), 1, 2, barrier_all, None, "dp")
        tf = _teacher_forced_parity(e1, pr1, primary["tokens"]) if rank == 0 and args.sampling == "greedy" else None
        e1.close()
        (dms, dwall), (dtok, ntok) = reduce_over_ranks([r1["dec_ms"], r1["wall"]], [r1["dec_tok"], r1["n_tok"]], "cuda")
        dp_leg = {"value": dtok / (dms * 1e-3), "unit": "tokens/s", "scaling": "weak",
                  "job_output_tokens_per_s": ntok / dwall, "jobs_timed": 2,
                  "parallelism": f"dp{world} (independent replicas, no data-path collective)"}
        if rank == 0:
            ref, got = r1["tokens"], primary["tokens"]
            same_prefix = sum(next((k for k, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
                              for a, b in zip(ref, got))
            total = sum(len(a) for a in ref)
            parity = {"teacher_forced": tf,
                      "free_running": {"identical_requests": sum(1 for a, b in zip(ref, got) if a == b),
                                       "requests": len(ref), "matching_prefix_tokens": same_prefix, "total_tokens": total},
                      "note": "in this run, same weights and prompts.  teacher_forced: every token the tensor-parallel engine "
                              "generated is scored by a single-GPU engine given the same prefix (prompt-logprob pass): it "
                              "must be that engine's argmax or lose to it by a few bf16 ulps of the logits (0.031 at |x| in "
                              "[4, 8)).  free_running: the two greedy continuations part ways at the first such near-tie -- "
                              "on this synthetic checkpoint many steps are <= 1-ulp races"}
        # (b) BASELINE configs[4]: Llama-3-70B TP=8, 256 concurrent requests
        if do_cfg4:
            B70 = 256
            e70, c70 = _build_engine("llama3-70b", max_seqs=B70, max_len=max_len, kv_tokens=B70 * (P + G + 32),
                                     max_batched=args.max_batched_tokens, tp=tp, rank=rank, local=local, weight_seed=77,
                                     layers=args.layers)
            log("70B engine built")
            if rank != 0:
                e70.worker_run()
                e70.close()
            else:
                p70 = prompts_for(c70, B70, 99)
                r = _timed_jobs(e70, p70, _sampling("greedy", G), 1, 2, barrier_local, None, "cfg[4]")
                pr = _profiled_pass(e70, p70)
                by = _step_bytes(c70, B70, P + G / 2, tp)
                sm = r["dec_ms"] / max(r["dec_steps"], 1)
                named70 = {"config": f"BASELINE.json configs[4]: llama3-70b bf16 TP={tp}, 256 concurrent requests, "
                                     f"512-in/128-out, greedy" + (f" (ONLY {args.layers} layers: code-path check)" if args.layers else ""),
                           "decode_tokens_per_s": r["dec_tok"] / (r["dec_ms"] * 1e-3),
                           "job_output_tokens_per_s": r["n_tok"] / r["wall"], "decode_step_ms": sm,
                           "ttft_p50_ms": 1e3 * statistics.median(r["ttfts"]),
                           "decode_step_algorithmic_bytes_per_gpu": by,
                           "decode_step_frac_of_hbm_roofline": by / (sm * 1e-3) / 1e9 / peaks()[0] if sm else None,
                           "exchange_ms_per_step": pr["exchange_ms"] / max(pr["decode_steps"], 1),
                           "exchanges_per_step": pr["exchange_calls"] / max(pr["decode_steps"], 1),
                           "gemm_ms_per_step": pr["gemm_ms"] / max(pr["decode_steps"], 1), "jobs_timed": 2}
                log(f"cfg[4] leg done: {named70['decode_tokens_per_s']:.0f} tok/s")
                e70.close()
            dist.barrier()

    # ============================================================ reduce + report
    if tp == 1:
        (dec_ms_m, decode_wall_m, wall_m), (dec_tok_s, n_tok_s, launches_s, n_tok_dec_s) = reduce_over_ranks(
            [primary["dec_ms"], primary["decode_wall"], primary["wall"]],
            [primary["dec_tok"], primary["n_tok"], primary["launches"], primary["n_tok_dec"]],
            "cuda" if world > 1 else "cpu")
    elif rank == 0:   # one engine: rank 0 holds the whole-job numbers (its step times include every exchange)
        dec_ms_m, decode_wall_m, wall_m = primary["dec_ms"], primary["decode_wall"], primary["wall"]
        dec_tok_s, n_tok_s, launches_s, n_tok_dec_s = (primary["dec_tok"], primary["n_tok"], primary["launches"],
                                                      primary["n_tok_dec"])
    if world > 1:
        dist.destroy_process_group()
    if rank != 0:
        return None
    peak, peak_src = peaks()
    bytes_step = _step_bytes(cfg, B, P + G / 2, tp)
    step_ms = primary["dec_ms"] / max(primary["dec_steps"], 1)
    gemm_ms, gemm_bytes, gemm_calls = prof["gemm_ms"], prof["gemm_bytes"], prof["gemm_calls"]
    achieved = gemm_bytes / (gemm_ms * 1e-3) / 1e9 if gemm_ms > 0 else None
    ttft_p50 = 1e3 * statistics.median(primary["ttfts"])
    out = {
        "metric": METRIC,
        "value": dec_tok_s / (dec_ms_m * 1e-3), "unit": "tokens/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1e3 * wall_m / args.steps, "higher_is_better": True,
        "scaling": "strong" if tp > 1 else "weak",
        "vs_baseline": None, "dtype": "bf16", "data": "synthetic (seeded N(0,0.02) weights, uniform random prompts)",
        "ttft_p50_ms": ttft_p50, "job_output_tokens_per_s": n_tok_s / wall_m,
        "config": {"workload": f"{args.model} bf16, {B} concurrent requests{'/GPU' if tp == 1 and world > 1 else ''}, "
                               f"{P}-in/{G}-out, {args.sampling} (BASELINE.json "
                               + ("configs[1])" if args.model == "llama3-8b" and B == 32 and args.sampling == "greedy" else
                                  "configs[0]: the 125m-class single greedy request)" if B == 1 and args.model in ("125m", "opt-125m")
                                  else "configs[2])" if args.model == "llama3-8b" and B == 64 and args.sampling == "cfg3"
                                  else "shape, not a named config)"),
                   "batch": B, "prompt_len": P, "gen_len": G,
                   "parallelism": (f"tp{tp} (ONE engine over {tp} GPUs: column-parallel qkv/gate_up, row-parallel o/down "
                                   f"with a fused push all-reduce + residual + RMSNorm kernel over NVLink peer memory, "
                                   f"vocab-parallel lm_head; CUDA-graph decode steps)"
                                   if tp > 1 else f"dp{world} (independent replicas, no collective)"),
                   "scheduler": f"continuous batching, chunked prefill, {args.max_batched_tokens} tokens per step",
                   "l2": "inputs larger than L2 (15 GB of weights streamed per decode step)",
                   "timing": "value: CUDA events on the engine stream over pure-decode steps; e2e: wall clock"},
        "e2e": {"value": n_tok_dec_s / decode_wall_m if decode_wall_m > 0 else None,
                "unit": "tokens/s", "h2d_bytes_per_step": primary["h2d"], "d2h_bytes_per_step": primary["d2h"],
                "job_output_tokens_per_s": n_tok_s / wall_m, "ttft_p50_ms": ttft_p50,
                "ttft_max_ms": 1e3 * max(primary["ttfts"]),
                "note": "through the C ABI with host buffers: add_request/run_until_idle/poll; value = tokens stamped after "
                        "the last request's first token / wall clock from that moment to the end of the job (decode "
                        "phase); job_output_tokens_per_s = all output tokens / whole-job wall clock incl. prefill"},
        "gpu_launches": int(launches_s),
        "graph_launches": int(primary["graph_launches"]),
        "clocks": primary["clocks"],
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s",
                     "frac": (achieved / peak) if achieved else None, "peak_source": peak_src,
                     "kernel": "gemm_bf16_wgmma_kernel", "launches_timed": int(gemm_calls),
                     "algorithmic_bytes_per_launch": gemm_bytes / max(gemm_calls, 1),
                     "avg_launch_us": 1e3 * gemm_ms / max(gemm_calls, 1),
                     "decode_step_ms": step_ms, "decode_step_algorithmic_bytes": bytes_step,
                     "decode_step_frac_of_hbm_roofline": bytes_step / (step_ms * 1e-3) / 1e9 / peak if step_ms else None},
    }
    if tp > 1:
        out["roofline"]["exchange_ms_per_step"] = prof["exchange_ms"] / max(prof["decode_steps"], 1)
        out["roofline"]["exchanges_per_step"] = prof["exchange_calls"] / max(prof["decode_steps"], 1)
        out["roofline"]["gemm_ms_per_step"] = prof["gemm_ms"] / max(prof["decode_steps"], 1)
        out["tp_parity"] = parity
        out["dp"] = dp_leg
        out["named_configs"] = {k: v for k, v in (("configs[3]", named), ("configs[4]", named70)) if v}
    return out


def main():
    args = parse_args()
    if args.dump_outputs and args.steps < 1:
        raise SystemExit("--dump-outputs needs at least one timed step")
    if args.dump_outputs and args.impl == "reference":
        raise SystemExit("--dump-outputs writes the GPU engine's outputs; --impl reference has none")
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.impl == "reference":
        if rank != 0:
            return
        # each bench step = one batched CPU decode step (bounded sample); --steps / --warmup are honoured as given
        ref = cpu_reference(args, args.steps, args.warmup, budget_s=240.0)
        print(json.dumps({
            "impl": "reference", "metric": METRIC,
            "value": ref["value"], "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            # wall time of one timed bench step (= one sampled CPU decode step); the full-depth step the value is
            # extrapolated to is full_depth_ms_per_step
            "ms_per_step": ref["sample_ms_per_step"], "full_depth_ms_per_step": ref["ms_per_step"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16", "data": "synthetic",
            "ttft_p50_ms": ref["ttft_p50_est_ms"],
            "config": {"workload": f"{args.model} bf16, {args.batch} concurrent requests, {args.prompt_len}-in, "
                                   f"decode steps on host cores (bounded sample, see cpu_baseline.sample)"},
            "cpu_baseline": {k: ref[k] for k in ("value", "unit", "cores", "kind", "sample")},
            "e2e": {"value": ref["value"], "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}), flush=True)
        return
    out = run_ours(args)
    if out is None:
        return
    if not args.no_cpu_baseline:   # rank 0, every N
        ref = cpu_reference(args, steps=args.cpu_steps, warmup=3, budget_s=args.cpu_budget_s)
        out["cpu_baseline"] = {k: ref[k] for k in ("value", "unit", "cores", "kind", "sample", "ttft_p50_est_ms")}
    else:
        out["cpu_baseline"] = None
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
