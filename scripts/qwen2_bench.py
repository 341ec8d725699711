"""The kernel-level costs of serving Qwen2 / Qwen2.5, through the C ABI, in one run:

  groups  decode attention at GQA groups 4, 5, 6, 7 and 8 over 8 kv heads (the same KV bytes for every group; Q read and
          O written grow with the group), at batch 32 and 256, contexts 512 / 2048 / 8192, head dims 128 and 64
          (tgis_k_attention_bench_hd, rotating over enough cache copies that a launch streams from HBM, not L2).
          Bytes = K and V tiles read (whole 32-token blocks) + Q read + O written.
  writer  the plain RoPE + KV writer (bf16 qkv in place) against the qkv-bias writer (fp32 accumulators + bias in, bf16
          qkv out) at Qwen2.5-7B heads (28 q, 4 kv, 128 dims), for T tokens.  Bytes: what each must move (see
          writer_bytes); at small T both fit in the 50 MB L2, so those rates are L2 rates.
  gemm    the qkv projection at the Qwen2.5-7B shape (N = 4608, K = 3584) with a bf16 and with an fp32 output, for T
          tokens (tgis_k_gemm): the price of the fp32 round trip the bias writer needs.

Every figure is the median over `--reps` alternating rounds of CUDA events around back-to-back launches.  The card's
name, power limit and SM clock are read in the same run and printed first; then one JSON line per measurement.  Needs a
GPU: there is no fallback.

  python scripts/qwen2_bench.py [--out qwen2_bench.json]
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
NKV, BLK = 8, 32


def attention_rows(reps: int):
    for hd in (128, 64):
        for batch in (32, 256):
            for ctx in (512, 2048, 8192):
                nblk = (ctx + BLK - 1) // BLK
                n_blocks = batch * nblk
                layer_elems = n_blocks * NKV * BLK * hd
                n_layers = max(2, int(400e6 // (layer_elems * 2 * 2)) + 1)
                kc = torch.randn(n_layers * layer_elems, device="cuda", dtype=torch.bfloat16)
                vc = torch.randn(n_layers * layer_elems, device="cuda", dtype=torch.bfloat16)
                bt = np.random.default_rng(0).permutation(n_blocks).astype(np.int32)
                seqs = np.array([[i, 1, ctx, i] for i in range(batch)], dtype=np.int32).reshape(-1)
                t = {G: [] for G in (4, 5, 6, 7, 8)}
                bufs = {G: (torch.randn(batch, (NKV * G + 2 * NKV) * hd, device="cuda", dtype=torch.bfloat16),
                            torch.empty(batch, NKV * G * hd, device="cuda", dtype=torch.bfloat16)) for G in t}
                kv_bytes = n_blocks * BLK * NKV * hd * 2 * 2
                iters = int(min(5000, max(50, 0.25 / (kv_bytes / (PEAK_GBPS * 1e9)))))
                for _ in range(reps):
                    for G in t:
                        qkv, out = bufs[G]
                        us = C.c_float(0)
                        rc = g.lib().tgis_k_attention_bench_hd(hd, g.ptr(qkv), g.ptr(kc), g.ptr(vc), g.i32p(seqs), batch,
                                                               g.i32p(bt), batch, nblk, g.ptr(out), NKV * G, NKV,
                                                               C.c_float(hd ** -0.5), n_layers,
                                                               C.c_int64(layer_elems * 2), iters, C.byref(us))
                        assert rc == 0, g.kerr()
                        t[G].append(us.value)
                for G, ts in t.items():
                    us = statistics.median(ts)
                    b = kv_bytes + batch * NKV * G * hd * 2 * 2
                    yield {"bench": "groups", "head_dim": hd, "group": G, "n_q": NKV * G, "n_kv": NKV, "batch": batch,
                           "kv_len": ctx, "us": round(us, 2), "us_all": [round(x, 2) for x in ts],
                           "GBps": round(b / us / 1e3, 1), "share_of_3.35TBps": round(b / us / 1e3 / PEAK_GBPS, 3)}
                del kc, vc, bufs
                torch.cuda.empty_cache()


def writer_bytes(T: int, n_q: int, n_kv: int, bias: bool) -> int:
    row = 128 * 2
    nh = n_q + 2 * n_kv
    if bias:   # fp32 acc read, bf16 qkv written (every head), bias read once per CTA row (counted once)
        qkv = T * nh * 128 * 4 + T * nh * row + nh * row
    else:      # q, k read + written; v read
        qkv = T * ((n_q + n_kv) * 2 + n_kv) * row
    return qkv + T * 2 * n_kv * row + T * (4 + 4 + row)


def writer_rows(reps: int, iters: int):
    n_q, n_kv = 28, 4
    nh = n_q + 2 * n_kv
    lib = g.lib()
    for T in (32, 256, 2048, 8192):
        gen = torch.Generator(device="cuda").manual_seed(T)
        acc = torch.randn(T, nh * 128, device="cuda", generator=gen)
        bias = torch.randn(nh * 128, device="cuda", generator=gen).bfloat16()
        qkv = acc.bfloat16()
        table = (torch.rand(8192, 128, device="cuda", generator=gen) * 2 - 1).bfloat16()
        rs = np.random.RandomState(T)
        pos = rs.randint(0, 8192, size=T).astype(np.int32)
        n_blocks = (T + 31) // 32
        slots = rs.permutation(n_blocks * 32)[:T].astype(np.int32)
        kc = torch.zeros(n_blocks, n_kv, 16, 32, 8, dtype=torch.bfloat16, device="cuda")
        vc = torch.zeros_like(kc)

        def run(b: bool, n: int) -> float:
            us = C.c_float(0)
            if b:
                rc = lib.tgis_k_rope_kv_bias(128, g.ptr(acc), g.ptr(bias), g.ptr(qkv), g.i32p(pos), g.i32p(slots),
                                             g.ptr(table), g.ptr(kc), g.ptr(vc), T, n_q, n_kv, n, C.byref(us))
            else:
                rc = lib.tgis_k_rope_kv_qknorm(g.ptr(qkv), g.i32p(pos), g.i32p(slots), g.ptr(table), g.ptr(kc),
                                               g.ptr(vc), T, n_q, n_kv, None, None, 0.0, n, C.byref(us))
            assert rc == 0, g.kerr()
            return us.value

        run(False, 50), run(True, 50)
        t = {False: [], True: []}
        for _ in range(reps):
            for b in (False, True):
                t[b].append(run(b, iters))
        row = {"bench": "writer", "heads": [n_q, n_kv], "T": T,
               "l2_resident": writer_bytes(T, n_q, n_kv, True) < 40e6}
        for b, name in ((False, "plain"), (True, "bias")):
            us = float(np.median(t[b]))
            nb = writer_bytes(T, n_q, n_kv, b)
            row[name] = {"us": round(us, 3), "per_rep_us": [round(x, 3) for x in t[b]], "bytes": nb,
                         "TB_per_s": round(nb / us / 1e6, 3)}
        row["bias_over_plain_us"] = round(row["bias"]["us"] - row["plain"]["us"], 3)
        yield row


def gemm_rows(reps: int):
    N, K = 4608, 3584
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    for T in (32, 512, 8192):
        x = torch.randn(max(T, 256), K, device="cuda").bfloat16()
        y = torch.empty(T, N, device="cuda", dtype=torch.float32)
        iters = 2000 if T <= 512 else 200
        t = {0: [], 1: []}
        for _ in range(reps):
            for f32 in (0, 1):
                ms = C.c_float(0)
                rc = g.lib().tgis_k_gemm(g.ptr(x), g.ptr(w), g.ptr(y), T, N, K, x.shape[0], 0, iters, C.byref(ms), f32)
                assert rc == 0, g.kerr()
                t[f32].append(ms.value * 1e3)
        row = {"bench": "gemm", "N": N, "K": K, "T": T}
        for f32, name in ((0, "bf16_out"), (1, "fp32_out")):
            row[name] = {"us": round(statistics.median(t[f32]), 2), "per_rep_us": [round(v, 2) for v in t[f32]]}
        row["fp32_over_bf16_us"] = round(row["fp32_out"]["us"] - row["bf16_out"]["us"], 2)
        row["extra_bytes"] = T * N * 2
        yield row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, metavar="FILE")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", nargs="+", default=["groups", "writer", "gemm"])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures GPU kernels: no GPU, no numbers"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    rows = []
    gens = {"groups": lambda: attention_rows(args.reps), "writer": lambda: writer_rows(args.reps, 2000),
            "gemm": lambda: gemm_rows(args.reps)}
    for name in args.only:
        for row in gens[name]():
            rows.append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        Path(args.out).write_text(json.dumps({"card": card, "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
