#!/bin/bash
# ncu --set full captures of the hot-path kernels (one GPU).  Reports are converted to raw CSV on the box (the .ncu-rep
# files are large); scripts/summarize_ncu_csv.py trims them into profiles/r02_ncu_*.csv.
cd "$(dirname "$0")/.."
mkdir -p gpurun_out/ncu
NCU="ncu --set full --clock-control none --import-source on -f"
run() {  # name, kernel regex, skip, count, command...
  name=$1; k=$2; s=$3; c=$4; shift 4
  timeout 400 $NCU -k "regex:$k" -s $s -c $c -o gpurun_out/ncu/$name "$@" > gpurun_out/ncu/$name.log 2>&1
  echo "ncu $name rc=$?"
  ncu -i gpurun_out/ncu/$name.ncu-rep --page raw --csv > gpurun_out/ncu/$name.csv 2>/dev/null
  rm -f gpurun_out/ncu/$name.ncu-rep
}
# decode step of a 2-layer 8B-shaped model, batch 32, context 512 (graphs off: ncu profiles plain launches)
run gemm_decode  "wgmma_kernel<32>"     9 9  python scripts/profile_decode.py 2 32 512 4 0
run attn_decode  "attn_decode"          2 2  python scripts/profile_decode.py 2 32 512 4 0
run norm         "rmsnorm_kernel"       10 2 python scripts/profile_decode.py 2 32 512 4 0
run sampler_greedy "tgis_sampler"       1 1  python scripts/profile_decode.py 2 32 512 4 0
run prefill_misc "rope_kvwrite|attn_prefill" 0 4 python scripts/profile_decode.py 2 32 512 2 0
SAMPLER_BENCH_ONLY="64:cfg3" run sampler_cfg3 "tgis_sampler" 1 1 python scripts/sampler_bench.py
# launch list of one decode step (shares, not absolutes)
timeout 400 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/ncu/launches.csv python scripts/profile_decode.py 4 32 512 6 0 > gpurun_out/ncu/launches.log 2>&1
echo "launch list rc=$?"
ls -la gpurun_out/ncu | head -20
