"""Prefix caching on the GPU: what a cache hit saves, and what the bookkeeping costs.

  1. Prefill attention of the warm shape (Llama-3-8B heads 32 / 8, a 64-token suffix over a P-token cached prefix,
     S such sequences in one launch): existing prefill kernel (mode 0) vs split-context cluster kernel (mode 1), device
     microseconds per layer (tgis_k_attention_split_bench).
  2. Engine, Llama-3-8B dims with synthetic weights: N requests that share a P-token prefix, each with a unique 64-token
     suffix, served one at a time after one warm-up request.  TTFT p50 / p90 with caching off vs on.
  3. Cold prompts (no shared prefix) of the same length, caching off vs on: the cost of the bookkeeping.

Writes one JSON document to stdout and to --out.  Needs an H100; there is no CPU path.
    python scripts/prefix_cache_bench.py --prefix 1024 4096 --n 32 --out /tmp/prefix_cache_bench.json
"""
from __future__ import annotations

import argparse
import ctypes as C
import dataclasses
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def gpu_info() -> dict:
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi failed: {e}"
    return {"nvidia_smi": out}


def attention_us(prefixes, suffixes, n_seqs_list, iters):
    import torch

    import tgis_gpu_utils as g
    from test_attention_precision_gpu import SCALE, Case

    res = []
    for P, suffix, S in [(p, q, s) for p in prefixes for q in suffixes for s in n_seqs_list]:
        case = Case(g, 32, 8, [(P, suffix, "rand")] * S, seed=P + S)
        row = {"prefix": P, "suffix": suffix, "seqs": S}
        outs = {}
        for mode in (0, 1):
            us = C.c_float(0)
            out = torch.zeros(case.q.shape, dtype=torch.bfloat16, device="cuda")
            rc = g.lib().tgis_k_attention_split_bench(
                g.ptr(case.qkv), g.ptr(case.kc), g.ptr(case.vc), g.i32p(case.seqs.reshape(-1)), S,
                g.i32p(case.bt.reshape(-1)), S, case.bt_stride, g.ptr(out), 32, 8, SCALE, mode, iters, C.byref(us))
            assert rc == 0, g.kerr()
            row[f"mode{mode}_us"] = round(us.value, 2)
            outs[mode] = out
        ref, _ = case.reference()
        n_bad, exact, _ = g.attention_bar(outs[1], ref, None)
        row["mode1_over_bar"], row["mode1_bit_exact"] = n_bad, round(exact, 4)
        res.append(row)
        print(json.dumps(row), flush=True)
    return res


def ttft_runs(prefixes, n, suffix, kv_tokens):
    import bench
    from vllm_tgis_adapter_b200.engine.core import make_sampling_params

    sp = make_sampling_params(greedy=True, max_tokens=1, min_tokens=1, eos_token_id=-1)
    vocab = 128256

    def ttft(eng, prompt):
        recs = eng.generate_sync([prompt], sp)[0]
        r = next(r for r in recs if r.new_token is not None)
        return (r.ts_first_token - r.ts_arrival) * 1e3, r.new_token

    res = []
    from vllm_tgis_adapter_b200.engine.core import PRESETS, NativeEngine

    cfg = dataclasses.replace(PRESETS["llama3-8b"], max_model_len=8192)
    kv_bytes = int((kv_tokens // 32 + 64) * 2 * cfg.n_layers * cfg.n_kv_heads * 32 * 128 * 2)
    for caching in (False, True):
        eng = NativeEngine(cfg, max_num_seqs=32, max_batched_tokens=8192, kv_cache_bytes=kv_bytes, seed=1234,
                           enable_prefix_caching=caching)
        bench._load_synthetic(eng, cfg, 0)   # bench.py's seeded on-device weights (read only, not modified)
        for P in prefixes:
            rng = np.random.RandomState(P)
            prefix = rng.randint(1000, vocab - 1000, size=P).tolist()
            warm = prefix + rng.randint(1000, vocab - 1000, size=suffix).tolist()
            ttft(eng, warm)   # warm-up: first launches of every shape, and (caching on) the prefix enters the cache
            shared, toks = [], []
            for i in range(n):
                t, tok = ttft(eng, prefix + rng.randint(1000, vocab - 1000, size=suffix).tolist())
                shared.append(t)
                toks.append(tok)
            cold = [ttft(eng, rng.randint(1000, vocab - 1000, size=P + suffix).tolist())[0] for _ in range(n // 2)]
            q, h, cached = eng.prefix_cache_stats()
            row = {"caching": caching, "prefix": P, "suffix": suffix, "n": n,
                   "shared_ttft_ms_p50": round(float(np.percentile(shared, 50)), 3),
                   "shared_ttft_ms_p90": round(float(np.percentile(shared, 90)), 3),
                   "cold_ttft_ms_p50": round(float(np.percentile(cold, 50)), 3),
                   "cold_ttft_ms_p90": round(float(np.percentile(cold, 90)), 3),
                   "first_tokens": toks[:8], "cache_queried_tokens": q, "cache_hit_tokens": h}
            res.append(row)
            print(json.dumps(row), flush=True)
        eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prefix", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--suffix", type=int, nargs="+", default=[64], help="query rows; the engine leg uses the first")
    ap.add_argument("--attn-prefix", type=int, nargs="+", default=None, help="contexts of the attention leg")
    ap.add_argument("--n", type=int, default=32)
    ap.add_argument("--seqs", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--skip-engine", action="store_true")
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    doc = {"gpu": gpu_info(), "attention": attention_us(a.attn_prefix or a.prefix, a.suffix, a.seqs, a.iters)}
    if not a.skip_engine:
        doc["engine"] = ttft_runs(a.prefix, a.n, a.suffix[0], kv_tokens=max(a.prefix) * 4 + 16384)
    doc["gpu_after"] = gpu_info()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(text)


if __name__ == "__main__":
    main()
