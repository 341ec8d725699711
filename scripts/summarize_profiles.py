"""Turn the scratch artefacts of a GPU run (gpurun_out/) into the small, tracked summaries under profiles/.
Usage: python scripts/summarize_profiles.py r01"""
import collections
import csv
import io
import json
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
SRC, DST = ROOT / "gpurun_out", ROOT / "profiles"
tag = sys.argv[1] if len(sys.argv) > 1 else "r01"
DST.mkdir(exist_ok=True)

KEYS = ["Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "lts__t_sector_hit_rate.pct", "smsp__inst_executed_pipe_uniform.sum", "sm__inst_executed_pipe_tensor.sum"]


def ncu_raw(rep: Path, out: Path) -> None:
    if not rep.exists():
        return
    r = subprocess.run(["ncu", "-i", str(rep), "--page", "raw", "--csv"], capture_output=True, text=True)
    rows = list(csv.reader(io.StringIO(r.stdout)))
    if len(rows) < 3:
        return
    hdr, units = rows[0], rows[1]
    idx = [i for i, h in enumerate(hdr) if h in KEYS]
    with out.open("w", newline="") as f:
        w = csv.writer(f)
        w.writerow([hdr[i] + (f" [{units[i]}]" if units[i] else "") for i in idx])
        for row in rows[2:]:
            w.writerow([row[i] for i in idx])


def launch_list(src: Path, out_agg: Path, out_raw: Path) -> None:
    if not src.exists():
        return
    lines = [l for l in src.read_text().splitlines() if not l.startswith("==")]
    rows = list(csv.DictReader(lines))
    order = []
    for row in rows:
        v = float(row["Metric Value"].replace(",", ""))
        v = v / 1e3 if row["Metric Unit"] == "ns" else v * 1e3 if row["Metric Unit"] == "ms" else v
        order.append((row["Kernel Name"].replace("void ", "").replace("tgis::", "").split("(")[0], row.get("Grid Size", ""), v))
    starts = [i for i, o in enumerate(order) if o[0].startswith("bitmap_set")]
    last = order[starts[-1]:] if starts else order
    agg = collections.OrderedDict()
    for n, g, v in last:
        a = agg.setdefault((n, g), [0, 0.0])
        a[0] += 1
        a[1] += v
    tot = sum(v for _, _, v in last)
    with out_agg.open("w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["kernel", "grid", "launches_in_step", "total_us", "avg_us", "share_of_step"])
        for (n, g), (c, v) in agg.items():
            w.writerow([n, g, c, f"{v:.1f}", f"{v / c:.1f}", f"{v / tot:.3f}"])
        w.writerow(["TOTAL (last decode step, ncu-serialised, cold caches: compare SHARES)", "", len(last), f"{tot:.1f}", "", "1.000"])
    with out_raw.open("w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["kernel", "grid", "gpu__time_duration_us"])
        for n, g, v in last:
            w.writerow([n, g, f"{v:.2f}"])


launch_list(SRC / "launches.csv", DST / f"{tag}_launches_decode_step_summary.csv", DST / f"{tag}_launches_decode_step.csv")
ncu_raw(SRC / "prof_attn.ncu-rep", DST / f"{tag}_ncu_full_attn_decode.csv")
ncu_raw(SRC / "prof_gemm_prefill.ncu-rep", DST / f"{tag}_ncu_full_gemm_prefill.csv")
for name in ("bench.log", "bench_ref.log", "parity_stats.json", "gemm_bench.json", "gemm_cta_sweep.json", "gemm_timeline.log",
             "gpu_info.txt", "tp2.log", "bench_tp2.log", "bench_tp4.log", "bench_dp2.log", "attn_bench.json", "grpc_bench.log",
             "bench_b64.log", "bench_b128.log", "bench_b256.log", "bench_b64_cfg3.log"):
    p = SRC / name
    if p.exists() and p.stat().st_size:
        shutil.copy(p, DST / f"{tag}_{name}")
print(sorted(x.name for x in DST.iterdir()))
