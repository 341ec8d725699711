"""Cost of Qwen3's per-head q / k RMSNorm inside the RoPE + KV writer: the plain writer (rope_kvwrite_kernel<128>) and the
QKNORM one (rope_kvwrite_kernel<128, true>) at Qwen3-8B heads (32 q, 8 kv, 128 dims), alternated, for T tokens.

Each figure is CUDA events around `iters` back-to-back launches on one stream (tgis_k_rope_kv_qknorm), the median of
`reps` alternating rounds.  Bytes per launch, what the writer must move: qkv rows of the q and k heads read and written
back, v heads read, K and V rows written to the cache, plus the positions / slot ids and the cos | sin rows it reads
(the QKNORM writer also reads its 2 x 128 weights per CTA, counted once).  Rate = bytes / time, against the H100 SXM's
3.35 TB/s.  Prints one JSON line with the card's name and power limit.

  python scripts/qk_norm_bench.py
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vllm_tgis_adapter_b200.engine import _lib  # noqa: E402

HBM_TBPS = 3.35


def writer_bytes(T: int, n_q: int, n_kv: int, qknorm: bool) -> int:
    row = 128 * 2
    qkv = T * ((n_q + n_kv) * 2 + n_kv) * row        # q, k read + written; v read
    cache = T * 2 * n_kv * row                         # K and V rows
    return qkv + cache + T * (4 + 4 + row) + (2 * row if qknorm else 0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, nargs="+", default=[32, 256, 2048, 8192])
    ap.add_argument("--n-q", type=int, default=32)
    ap.add_argument("--n-kv", type=int, default=8)
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark times GPU kernels: no GPU, no numbers"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    lib = _lib.load_library()
    n_q, n_kv = args.n_q, args.n_kv
    nh = n_q + 2 * n_kv
    rows = []
    for T in args.tokens:
        gen = torch.Generator(device="cuda").manual_seed(T)
        qkv = torch.randn(T, nh, 128, device="cuda", generator=gen).bfloat16()
        table = (torch.rand(8192, 128, device="cuda", generator=gen) * 2 - 1).bfloat16()
        qn = (0.5 + torch.rand(128, device="cuda", generator=gen)).bfloat16()
        kn = (0.5 + torch.rand(128, device="cuda", generator=gen)).bfloat16()
        rs = np.random.RandomState(T)
        pos = rs.randint(0, 8192, size=T).astype(np.int32)
        n_blocks = (T + 31) // 32
        slots = rs.permutation(n_blocks * 32)[:T].astype(np.int32)
        kc = torch.zeros(n_blocks, n_kv, 16, 32, 8, dtype=torch.bfloat16, device="cuda")
        vc = torch.zeros_like(kc)
        ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))  # noqa: E731

        def run(norm: bool, iters: int) -> float:
            us = C.c_float(0)
            rc = lib.tgis_k_rope_kv_qknorm(C.c_void_p(qkv.data_ptr()), ip(pos), ip(slots), C.c_void_p(table.data_ptr()),
                                           C.c_void_p(kc.data_ptr()), C.c_void_p(vc.data_ptr()), T, n_q, n_kv,
                                           C.c_void_p(qn.data_ptr()) if norm else None,
                                           C.c_void_p(kn.data_ptr()) if norm else None, 1e-6, iters, C.byref(us))
            assert rc == 0, lib.tgis_k_last_error()
            return us.value

        run(False, 50), run(True, 50)          # warm-up: module load, clocks
        t = {False: [], True: []}
        for _ in range(args.reps):
            for norm in (False, True):
                t[norm].append(run(norm, args.iters))
        row = {"T": T}
        for norm, name in ((False, "plain"), (True, "qknorm")):
            us = float(np.median(t[norm]))
            b = writer_bytes(T, n_q, n_kv, norm)
            row[name] = {"us": round(us, 3), "per_rep_us": [round(x, 3) for x in t[norm]],
                         "TB_per_s": round(b / us / 1e6, 3), "share_of_3.35TBps": round(b / us / 1e6 / HBM_TBPS, 3)}
        row["qknorm_over_plain_us"] = round(row["qknorm"]["us"] - row["plain"]["us"], 3)
        rows.append(row)
    print(json.dumps({"card": card, "heads": [n_q, n_kv], "iters": args.iters, "rows": rows}), flush=True)


if __name__ == "__main__":
    main()
