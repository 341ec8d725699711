"""Sliding-window decode attention beside full attention, through the C ABI (tgis_k_attention_bench_window).

Mistral-7B heads (32 q / 8 kv heads of 128), batch 32, contexts 2048 .. 32768, window 4096 against window 0 (full
attention), alternating ROUNDS times.  Every timing is CUDA events around `iters` launches after two warm-up launches,
rotating over enough cache copies that a launch streams from HBM, not L2.  Bytes = the K and V tiles actually read (the
whole 32-token blocks from the one holding max(0, kv_len - window) to the last) + Q read + O written.  A windowed
launch reads at most W + 31 tokens of KV per sequence however long the context, so its time should stay flat beyond W.
The share of peak is against the H100 SXM data-sheet 3.35 TB/s; the card's name, power limit and clocks are read in the
same run and printed with the numbers, one JSON line per measurement.  Needs a GPU: there is no fallback.

  python scripts/swa_attn_bench.py [--out swa_attn_bench.json]
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

PEAK_GBPS = 3350.0   # H100 SXM data sheet, HBM3
NQ, NKV, HD, BLK, ROUNDS, BATCH, WINDOW = 32, 8, 128, 32, 3, 32, 4096


def traffic_bytes(batch: int, kv_len: int, window: int) -> int:
    lo = max(0, kv_len - window) if window else 0
    blocks = (kv_len - 1) // BLK - lo // BLK + 1
    kv = batch * blocks * BLK * NKV * HD * 2 * 2          # K and V, bf16, whole blocks
    q_o = batch * NQ * HD * 2 * 2                         # Q read, O written
    return kv + q_o


class Arm:
    def __init__(self, kv_len: int, window: int, cache: "Cache"):
        self.kv_len, self.window, self.c = kv_len, window, cache
        self.bytes = traffic_bytes(BATCH, kv_len, window)
        self.iters = int(min(5000, max(50, 0.25 / (self.bytes / (PEAK_GBPS * 1e9)))))
        self.us = []

    def run(self) -> None:
        c = self.c
        us = C.c_float(0)
        rc = g.lib().tgis_k_attention_bench_window(HD, g.ptr(c.qkv), g.ptr(c.kc), g.ptr(c.vc),
                                                   g.i32p(c.seqs.reshape(-1)), BATCH, g.i32p(c.bt.reshape(-1)), BATCH,
                                                   c.nblk_seq, g.ptr(c.out), NQ, NKV, C.c_float(HD ** -0.5),
                                                   c.n_layers, C.c_int64(c.layer_elems * 2), self.iters, C.byref(us),
                                                   self.window)
        assert rc == 0, g.kerr()
        self.us.append(us.value)

    def result(self) -> dict:
        us = statistics.median(self.us)
        gbps = self.bytes / us / 1e3
        return {"window": self.window, "batch": BATCH, "kv_len": self.kv_len, "bytes_read": self.bytes,
                "iters": self.iters, "us_median": us, "us_all": self.us, "GBps": gbps, "share_of_3.35TBps": gbps / PEAK_GBPS}


class Cache:
    """one paged cache for BATCH sequences of kv_len tokens, copied n_layers times"""

    def __init__(self, kv_len: int):
        self.nblk_seq = (kv_len + BLK - 1) // BLK
        n_blocks = BATCH * self.nblk_seq
        self.layer_elems = n_blocks * NKV * BLK * HD
        self.n_layers = max(2, int(400e6 // (self.layer_elems * 2 * 2)) + 1)
        self.kc = torch.randn(self.n_layers * self.layer_elems, device="cuda", dtype=torch.bfloat16)
        self.vc = torch.randn(self.n_layers * self.layer_elems, device="cuda", dtype=torch.bfloat16)
        self.qkv = torch.randn(BATCH, (NQ + 2 * NKV) * HD, device="cuda", dtype=torch.bfloat16)
        self.out = torch.empty(BATCH, NQ * HD, dtype=torch.bfloat16, device="cuda")
        self.bt = np.random.default_rng(0).permutation(n_blocks).astype(np.int32).reshape(BATCH, self.nblk_seq)
        self.seqs = np.array([[i, 1, kv_len, i] for i in range(BATCH)], dtype=np.int32)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, metavar="FILE", help="also write the card and every row to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU kernels: no GPU, no numbers"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    rows = []
    for ctx in (2048, 4096, 8192, 16384, 32768):
        cache = Cache(ctx)
        arms = [Arm(ctx, WINDOW, cache), Arm(ctx, 0, cache)]
        for _ in range(ROUNDS):
            for a in arms:
                a.run()
        for a in arms:
            rows.append(a.result())
            print(json.dumps(rows[-1]), flush=True)
        del cache, arms
        torch.cuda.empty_cache()
    if args.out:
        Path(args.out).write_text(json.dumps({"card": card, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
