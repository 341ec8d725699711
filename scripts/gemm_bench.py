"""Micro-benchmark of the wgmma GEMM through the C ABI on Llama-3-8B decode / prefill shapes.
Weights are rotated over several distinct buffers so every launch streams from HBM, not L2."""
import ctypes as C
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import tgis_gpu_utils as g  # noqa: E402

SHAPES = [("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336),
          ("lm_head", 128256, 4096)]
TS = (16, 32, 64, 128, 256, 2048, 8192)
if len(sys.argv) > 1 and sys.argv[1] == "tp":   # per-GPU shard shapes of the tensor-parallel named configs
    SHAPES = [("8b_tp4_qkv", 1536, 4096), ("8b_tp4_o", 4096, 1024), ("8b_tp4_gate_up", 7168, 4096), ("8b_tp4_down", 4096, 3584),
              ("70b_tp8_qkv", 1280, 8192), ("70b_tp8_o", 8192, 1024), ("70b_tp8_gate_up", 7168, 8192),
              ("70b_tp8_down", 8192, 3584), ("70b_tp8_lm_head", 16032, 8192)]
    TS = (32, 128, 256)
if len(sys.argv) > 1 and sys.argv[1] == "decode":   # quick A/B of the decode-shaped launches only
    TS = (32, 64, 128)
PEAK = 6566.7
res = []
for name, N, K in SHAPES:
    for T in TS:
        if name == "lm_head" and T > 256:
            continue
        n_buf = max(2, int(600e6 // (N * K * 2)) + 1) if T <= 256 else 1
        ws = [(torch.randn(N, K, device="cuda") * 0.02).bfloat16() for _ in range(n_buf)]
        rows = max(T, 256)
        x = (torch.randn(rows, K, device="cuda") * 0.5).bfloat16()
        y = torch.empty(T, N, dtype=torch.bfloat16, device="cuda")
        ms = C.c_float(0)
        # warm
        for w in ws:
            assert g.lib().tgis_k_gemm(g.ptr(x), g.ptr(w), g.ptr(y), T, N, K, rows, 0, 1, C.byref(ms), 0) == 0, g.kerr()
        tot, cnt = 0.0, 0
        for rep in range(3):
            for w in ws:
                assert g.lib().tgis_k_gemm(g.ptr(x), g.ptr(w), g.ptr(y), T, N, K, rows, 0, 1, C.byref(ms), 0) == 0
                tot += ms.value
                cnt += 1
        t = tot / cnt
        by = N * K * 2 + T * K * 2 + T * N * 2
        fl = 2.0 * T * N * K
        r = {"gemm": name, "T": T, "N": N, "K": K, "us": 1e3 * t, "GBps": by / t / 1e6, "hbm_frac": by / t / 1e6 / PEAK,
             "TFLOPs": fl / t / 1e9}
        res.append(r)
        print(json.dumps(r), flush=True)
        del ws, x, y
        torch.cuda.empty_cache()
Path("gpurun_out").mkdir(exist_ok=True)
Path(f"gpurun_out/gemm_bench_{sys.argv[1]}.json" if len(sys.argv) > 1 else "gpurun_out/gemm_bench.json").write_text(json.dumps(res, indent=1))
