"""Decode attention at 96-dim heads beside the 128- and 64-dim kernels at equal KV bytes, through the C ABI
(tgis_k_attention_bench_hd).

All three run 32 q / 8 kv heads (GQA group 4) at batch 32 and 256; D = 96 over contexts 512 / 2048 / 8192, D = 128 over
3/4 of those and D = 64 over 3/2, so every arm streams the same K / V bytes.  With --only96 the second arm is instead the
Phi-3-mini head layout (32 q / 32 kv heads of 96, group 1) at the D = 96 contexts, with 4x the bytes.  The arms alternate, ROUNDS times
each; every timing is CUDA events around `iters` launches after two warm-up launches, rotating over enough cache copies
that a launch streams from HBM, not L2.  Bytes = K and V tiles read (whole 32-token blocks) + Q read + O written,
computed from the shapes below.  The share of peak is against the H100 SXM data-sheet 3.35 TB/s; the card's name and
power limit are read in the same run and printed with the numbers, one JSON line per measurement (--out FILE also writes
them as one JSON document).  Set TGIS_ENGINE_LIB to time another build of the same sources (the decode ring at D = 96 is
-DTGIS_DEC_RING96=N, scripts/build_variant.py).  Needs a GPU: there is no fallback.

  python scripts/attn_hd96_bench.py [--out attn_hd96_bench.json] [--only96]
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
NQ, NKV, BLK, ROUNDS = 32, 8, 32, 3


def traffic_bytes(batch: int, kv_len: int, hd: int, nkv: int = NKV) -> int:
    blocks = (kv_len + BLK - 1) // BLK
    kv = batch * blocks * BLK * nkv * hd * 2 * 2          # K and V, bf16, whole blocks
    q_o = batch * NQ * hd * 2 * 2                         # Q read, O written
    return kv + q_o


class Arm:
    def __init__(self, hd: int, batch: int, kv_len: int, nkv: int = NKV):
        self.hd, self.batch, self.kv_len, self.nkv = hd, batch, kv_len, nkv
        self.nblk_seq = (kv_len + BLK - 1) // BLK
        n_blocks = batch * self.nblk_seq
        self.layer_elems = n_blocks * nkv * BLK * hd
        self.n_layers = max(2, int(400e6 // (self.layer_elems * 2 * 2)) + 1)
        self.kc = torch.randn(self.n_layers * self.layer_elems, device="cuda", dtype=torch.bfloat16)
        self.vc = torch.randn(self.n_layers * self.layer_elems, device="cuda", dtype=torch.bfloat16)
        self.qkv = torch.randn(batch, (NQ + 2 * nkv) * hd, device="cuda", dtype=torch.bfloat16)
        self.out = torch.empty(batch, NQ * hd, dtype=torch.bfloat16, device="cuda")
        self.bt = np.random.default_rng(0).permutation(n_blocks).astype(np.int32).reshape(batch, self.nblk_seq)
        self.seqs = np.array([[i, 1, kv_len, i] for i in range(batch)], dtype=np.int32)
        self.bytes = traffic_bytes(batch, kv_len, hd, nkv)
        self.iters = int(min(5000, max(50, 0.25 / (self.bytes / (PEAK_GBPS * 1e9)))))
        self.us = []

    def run(self) -> None:
        us = C.c_float(0)
        rc = g.lib().tgis_k_attention_bench_hd(self.hd, g.ptr(self.qkv), g.ptr(self.kc), g.ptr(self.vc),
                                               g.i32p(self.seqs.reshape(-1)), self.batch, g.i32p(self.bt.reshape(-1)),
                                               self.batch, self.nblk_seq, g.ptr(self.out), NQ, self.nkv,
                                               C.c_float(self.hd ** -0.5), self.n_layers,
                                               C.c_int64(self.layer_elems * 2), self.iters, C.byref(us))
        assert rc == 0, g.kerr()
        self.us.append(us.value)

    def result(self) -> dict:
        us = statistics.median(self.us)
        gbps = self.bytes / us / 1e3
        return {"head_dim": self.hd, "n_kv": self.nkv, "batch": self.batch, "kv_len": self.kv_len, "bytes": self.bytes, "iters": self.iters,
                "us_median": us, "us_all": self.us, "GBps": gbps, "share_of_3.35TBps": gbps / PEAK_GBPS}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, metavar="FILE", help="also write the card and every row to this JSON file")
    ap.add_argument("--only96", action="store_true", help="time D = 96 only: group 4 and Phi-3-mini's group 1")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU kernels: no GPU, no numbers"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    rows = []
    for batch in (32, 256):
        for ctx in (512, 2048, 8192):
            arms = [Arm(96, batch, ctx)]
            if args.only96:
                arms.append(Arm(96, batch, ctx, nkv=NQ))
            else:
                arms += [Arm(128, batch, ctx * 3 // 4), Arm(64, batch, ctx * 3 // 2)]
                assert all(abs(a.bytes - arms[0].bytes) <= batch * NQ * 128 * 4 for a in arms[1:])   # same KV bytes
            for _ in range(ROUNDS):
                for arm in arms:
                    arm.run()
            for arm in arms:
                rows.append(arm.result())
                print(json.dumps(rows[-1]), flush=True)
            del arms
            torch.cuda.empty_cache()
    if args.out:
        Path(args.out).write_text(json.dumps({"card": card, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
