"""Multi-query decode attention (48 q heads over 1 kv head: StarCoder-15B, Granite-20B/34B-Code) beside 48 over 8 (G = 6),
through the C ABI (tgis_k_attention_bench_window).

Both do the same query work; 48/1 reads 1/8 of the KV bytes, in head octets (6 work units per (sequence, split), each
streaming the split's K / V tiles, the later ones from L2).  Batch 32 and 256, contexts 512, 2048 and 8192, the two
arms alternating ROUNDS times, medians reported.  Every timing is CUDA events around `iters` launches after two warm-up
launches, rotating over enough cache copies that a launch streams from HBM, not L2.  Bytes = the K and V tiles of the
sequences (whole 32-token blocks, read once from HBM) + Q read + O written; MMA FLOPs = the m16n8k16 tiles issued (per
32-token block and unit: QK^T 2 x 8 and PV 2 x 8 x 2 (bf16 hi + lo), 4096 FLOPs each).  The bound that applies is the
larger of bytes / 3.35 TB/s and FLOPs / 989 TFLOP/s (H100 SXM data sheet; dense bf16); the card's name, power limit and
clocks are read in the same run and printed with the numbers, one JSON line per measurement.  Needs a GPU.

  python scripts/mqa_attn_bench.py [--out mqa_attn_bench.json]
"""
import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
import tgis_gpu_utils as g  # noqa: E402

PEAK_GBPS, PEAK_TFLOPS = 3350.0, 989.0
NQ, HD, BLK, ROUNDS = 48, 128, 32, 5


def traffic(batch: int, kv_len: int, n_kv: int) -> tuple[int, float]:
    blocks = (kv_len + BLK - 1) // BLK
    kv = batch * blocks * BLK * n_kv * HD * 2 * 2
    q_o = batch * NQ * HD * 2 * 2
    units = n_kv * ((NQ // n_kv + 7) // 8)                 # (kv head, octet) per (sequence, split)
    flops = batch * blocks * units * (16 + 32) * 4096.0
    return kv + q_o, flops


class Arm:
    def __init__(self, batch: int, kv_len: int, n_kv: int):
        self.batch, self.kv_len, self.n_kv = batch, kv_len, n_kv
        self.bytes, self.flops = traffic(batch, kv_len, n_kv)
        self.nblk_seq = (kv_len + BLK - 1) // BLK
        n_blocks = batch * self.nblk_seq
        self.layer_elems = n_blocks * n_kv * BLK * HD
        self.n_layers = max(2, int(400e6 // (self.layer_elems * 2 * 2)) + 1)
        self.kc = torch.randn(self.n_layers * self.layer_elems, device="cuda", dtype=torch.bfloat16)
        self.vc = torch.randn(self.n_layers * self.layer_elems, device="cuda", dtype=torch.bfloat16)
        self.qkv = torch.randn(batch, (NQ + 2 * n_kv) * HD, device="cuda", dtype=torch.bfloat16)
        self.out = torch.empty(batch, NQ * HD, dtype=torch.bfloat16, device="cuda")
        self.bt = np.random.default_rng(0).permutation(n_blocks).astype(np.int32).reshape(batch, self.nblk_seq)
        self.seqs = np.array([[i, 1, kv_len, i] for i in range(batch)], dtype=np.int32)
        self.iters = int(min(2000, max(30, 0.2 / max(self.bytes / (PEAK_GBPS * 1e9), 5e-6))))
        self.us = []

    def run(self) -> None:
        us = C.c_float(0)
        rc = g.lib().tgis_k_attention_bench_window(HD, g.ptr(self.qkv), g.ptr(self.kc), g.ptr(self.vc),
                                                   g.i32p(self.seqs.reshape(-1)), self.batch,
                                                   g.i32p(self.bt.reshape(-1)), self.batch, self.nblk_seq,
                                                   g.ptr(self.out), NQ, self.n_kv, C.c_float(HD ** -0.5),
                                                   self.n_layers, C.c_int64(self.layer_elems * 2), self.iters,
                                                   C.byref(us), 0)
        assert rc == 0, g.kerr()
        self.us.append(us.value)

    def result(self) -> dict:
        us = statistics.median(self.us)
        t_bytes, t_flops = self.bytes / (PEAK_GBPS * 1e3), self.flops / (PEAK_TFLOPS * 1e6)
        return {"n_q": NQ, "n_kv": self.n_kv, "batch": self.batch, "kv_len": self.kv_len, "bytes_read": self.bytes,
                "mma_flops": self.flops, "iters": self.iters, "us_median": us, "us_spread": [min(self.us), max(self.us)],
                "TBps": self.bytes / us / 1e6, "bound": "bytes" if t_bytes >= t_flops else "mma_flops",
                "share_of_bound": max(t_bytes, t_flops) / us}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, metavar="FILE", help="also write the card and every row to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU kernels: no GPU, no numbers"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    rows = []
    for batch in (32, 256):
        for ctx in (512, 2048, 8192):
            arms = [Arm(batch, ctx, 1), Arm(batch, ctx, 8)]
            for _ in range(ROUNDS):
                for a in arms:
                    a.run()
            res = [a.result() for a in arms]
            res[0]["speedup_vs_48_over_8"] = res[1]["us_median"] / res[0]["us_median"]
            for r in res:
                rows.append(r)
                print(json.dumps(r), flush=True)
            del arms
            torch.cuda.empty_cache()
    if args.out:
        Path(args.out).write_text(json.dumps({"card": card, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
