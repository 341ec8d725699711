"""Engine-level cost of the two late round-2 features on the BASELINE configs[1] shape (Llama-3-8B dims, 32 requests,
512-in / 64-out, greedy, one H100): device-timed decode ms per step (tgis_status.gpu_decode_ms / decode_steps) for
  base    : no adapter, no grammar (the fused production path, CUDA-graph decode steps)
  lora    : every request on ONE rank-16 adapter over all seven projections (unfused projections + lora.cu, graphs)
  lora4   : the requests spread over FOUR adapters (mixed-adapter token tiles)
  guided  : every request under a token bitmask (a provider that allows every token: the cost measured is the per-step
            host callback x 32, the 16 KB H2D per row and the masked sampler instantiation -- not a grammar's own cost)
Writes gpurun_out/feature_decode_bench.json."""
import ctypes as C
import json
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from vllm_tgis_adapter_b200.engine.core import PRESETS, NativeEngine, make_sampling_params  # noqa: E402
from vllm_tgis_adapter_b200.engine.guided import MASK_FN  # noqa: E402

B, P, G, R = 32, 512, 64, 16
layers = int(os.environ.get("FEATURE_BENCH_LAYERS", "32"))
import dataclasses  # noqa: E402

cfg = dataclasses.replace(PRESETS["llama3-8b"], max_model_len=P + G + 64, n_layers=layers)
blocks = (B * (P + G + 64)) // 32 + 2 * B
kv_bytes = int(blocks * 2 * cfg.n_layers * cfg.n_kv_heads * 32 * 128 * 2 * 1.1)
eng = NativeEngine(cfg, max_num_seqs=B, max_batched_tokens=2048, kv_cache_bytes=kv_bytes, seed=1, max_loras=4, max_lora_rank=R)
bench._load_synthetic(eng, cfg, 7)
g = torch.Generator(device="cuda").manual_seed(3)
q_dim, kv_dim = cfg.n_q_heads * 128, cfg.n_kv_heads * 128
shapes = {"q_proj": (cfg.hidden, q_dim), "k_proj": (cfg.hidden, kv_dim), "v_proj": (cfg.hidden, kv_dim),
          "o_proj": (q_dim, cfg.hidden), "gate_proj": (cfg.hidden, cfg.ffn), "up_proj": (cfg.hidden, cfg.ffn),
          "down_proj": (cfg.ffn, cfg.hidden)}
for slot in range(1, 5):
    w = {}
    for li in range(cfg.n_layers):
        for m, (fin, fout) in shapes.items():
            w[(li, m)] = ((torch.randn(R, fin, generator=g, device="cuda") * 0.01).to(torch.bfloat16),
                          (torch.randn(fout, R, generator=g, device="cuda") * 0.01).to(torch.bfloat16))
    eng.load_adapter(slot, w)
    del w
rng = np.random.RandomState(1234)
prompts = [rng.randint(1000, cfg.vocab - 1000, size=P).tolist() for _ in range(B)]
words = (cfg.vocab + 31) // 32


def allow_all(_user, _rid, _new, _n, bits, n_words):
    C.memset(bits, 0xFF, 4 * n_words)
    return 0


cb = MASK_FN(allow_all)
eng.set_mask_provider(cb)


def run(tag, slots, guided):
    res = None
    for it in range(2):   # first pass warms up (graph capture), second is reported
        st0 = eng.status()
        t0 = time.perf_counter()
        for i, pr in enumerate(prompts):
            eng.add_request(f"r{i}", pr, make_sampling_params(greedy=True, max_tokens=G, min_tokens=G, eos_token_id=2,
                                                             lora_slot=slots[i], guided=guided))
        eng.run_until_idle()
        wall = time.perf_counter() - t0
        while eng.poll(0):
            pass
        st1 = eng.status()
        steps = st1.decode_steps - st0.decode_steps
        res = {"case": tag, "decode_ms_per_step": (st1.gpu_decode_ms - st0.gpu_decode_ms) / max(steps, 1),
               "decode_steps": steps, "mixed_ms_total": st1.gpu_mixed_ms - st0.gpu_mixed_ms,
               "graph_launches": st1.graph_launches - st0.graph_launches,
               "kernel_launches_per_decode_step": None, "job_wall_s": wall, "layers": cfg.n_layers}
    print(json.dumps(res), flush=True)
    return res


out = [run("base", [0] * B, False), run("lora (1 adapter, rank 16, 7 modules)", [1] * B, False),
       run("lora4 (4 adapters mixed)", [1 + i % 4 for i in range(B)], False), run("guided (allow-all mask)", [0] * B, True)]
os.makedirs("gpurun_out", exist_ok=True)
Path("gpurun_out/feature_decode_bench.json").write_text(json.dumps(out, indent=1))
eng.close()
