#!/bin/bash
# One gpurun call: kernel parity tests, engine parity tests, (optionally) bench + profiles.  Everything is wrapped in
# `timeout` and logs into gpurun_out/ so a failure in one stage still returns the evidence of the others.
set -u
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,memory.total,clocks.max.sm,driver_version --format=csv > gpurun_out/gpu_info.txt 2>&1
nproc >> gpurun_out/gpu_info.txt; free -g | head -2 >> gpurun_out/gpu_info.txt
STAGES="${1:-kernels engine}"
NGPU="${NGPU:-2}"
for st in $STAGES; do
  case $st in
    kernels) timeout 900 python -m pytest tests/test_kernels_gpu.py -m gpu -q -x --no-header -p no:cacheprovider > gpurun_out/test_kernels.log 2>&1; echo "kernels rc=$?" ;;
    kernels_all) timeout 1200 python -m pytest tests/test_kernels_gpu.py -m gpu -q --no-header -p no:cacheprovider > gpurun_out/test_kernels.log 2>&1; echo "kernels rc=$?" ;;
    engine) timeout 900 python -m pytest tests/test_engine_gpu.py -m gpu -q --no-header -p no:cacheprovider > gpurun_out/test_engine.log 2>&1; echo "engine rc=$?" ;;
    all) timeout 1800 python -m pytest tests -m gpu -q --no-header -p no:cacheprovider > gpurun_out/test_all.log 2>&1; echo "all rc=$?" ;;
    smoke) timeout 600 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/smoke.log 2>&1; echo "smoke rc=$?" ;;
    bench) timeout 900 python bench.py > gpurun_out/bench.log 2> gpurun_out/bench.err; echo "bench rc=$?" ;;
    bench_small) timeout 300 python bench.py --model small --batch 8 --prompt-len 128 --gen-len 32 --no-cpu-baseline > gpurun_out/bench_small.log 2> gpurun_out/bench_small.err; echo "bench_small rc=$?" ;;
    bench_modes) for gr in 0 1; do TGIS_CUDA_GRAPHS=$gr timeout 400 python bench.py --no-cpu-baseline --steps 2 --warmup 3 > gpurun_out/bench_graph${gr}.log 2> gpurun_out/bench_graph${gr}.err; done; echo "bench_modes rc=$?" ;;
    bench_gpu) timeout 600 python bench.py --no-cpu-baseline > gpurun_out/bench_gpu.log 2> gpurun_out/bench_gpu.err; echo "bench_gpu rc=$?" ;;
    bench_ref) timeout 400 python bench.py --impl reference --steps 1 --warmup 1 > gpurun_out/bench_ref.log 2> gpurun_out/bench_ref.err; echo "bench_ref rc=$?" ;;
    prof_list) timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/launches.csv python scripts/profile_decode.py 4 32 512 6 0 > gpurun_out/prof_list.log 2>&1; echo "prof_list rc=$?" ;;
    prof_attn) timeout 900 ncu --set full --clock-control none --import-source on -k regex:attn_decode -s 2 -c 2 -f -o gpurun_out/prof_attn python scripts/profile_decode.py 2 32 512 4 0 > gpurun_out/prof_attn.log 2>&1; echo "prof_attn rc=$?" ;;
    decode_quick) for pdl in 0 1; do for gr in 0 1; do TGIS_PDL=$pdl timeout 300 python scripts/profile_decode.py 8 32 512 24 $gr > gpurun_out/decode_pdl${pdl}_graph${gr}.log 2>&1; done; done; echo "decode_quick rc=$?" ;;
    tp2) timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port 29511 scripts/tp_check.py tiny > gpurun_out/tp2.log 2>&1; echo "tp2 rc=$?"; timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node=2 --master-addr 127.0.0.1 --master-port 29512 scripts/tp_check.py tiny > gpurun_out/tp2_b.log 2>&1; echo "tp2 small rc=$?" ;;
    tpn) timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node=$NGPU --master-addr 127.0.0.1 --master-port 29513 scripts/tp_check.py tp8 > gpurun_out/tp${NGPU}_check.log 2>&1; echo "tpn rc=$?"; tail -2 gpurun_out/tp${NGPU}_check.log ;;
    tpserver) timeout 600 python scripts/tp_server_smoke.py $NGPU tiny > gpurun_out/tp_server_smoke.log 2>&1; echo "tpserver rc=$?"; tail -3 gpurun_out/tp_server_smoke.log ;;
    grpc_bench) timeout 600 python scripts/grpc_bench.py > gpurun_out/grpc_bench.log 2>&1; echo "grpc_bench rc=$?" ;;
    bench_tp) timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node=$NGPU --master-addr 127.0.0.1 --master-port 29541 bench.py --gpus $NGPU --parallel tp --no-cpu-baseline --steps 2 --warmup 3 > gpurun_out/bench_tp$NGPU.log 2> gpurun_out/bench_tp$NGPU.err; echo "bench_tp rc=$?" ;;
    bench_dp) timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node=$NGPU --master-addr 127.0.0.1 --master-port 29542 bench.py --gpus $NGPU --no-cpu-baseline --steps 2 --warmup 3 > gpurun_out/bench_dp$NGPU.log 2> gpurun_out/bench_dp$NGPU.err; echo "bench_dp rc=$?" ;;
    bench_batches) for b in 64 128 256; do timeout 400 python bench.py --no-cpu-baseline --steps 1 --warmup 3 --batch $b > gpurun_out/bench_b$b.log 2> gpurun_out/bench_b$b.err; done; timeout 400 python bench.py --no-cpu-baseline --steps 1 --warmup 3 --batch 64 --sampling cfg3 > gpurun_out/bench_b64_cfg3.log 2> gpurun_out/bench_b64_cfg3.err; echo "bench_batches rc=$?" ;;
    timeline) timeout 300 python scripts/gemm_timeline.py > gpurun_out/gemm_timeline.log 2>&1; echo "timeline rc=$?" ;;
    ctasweep) timeout 300 python scripts/gemm_cta_sweep.py > gpurun_out/gemm_cta_sweep.log 2>&1; echo "ctasweep rc=$?" ;;
    attnbench) timeout 300 python scripts/attn_bench.py > gpurun_out/attn_bench.log 2>&1; echo "attnbench rc=$?" ;;
    gemmbench) timeout 600 python scripts/gemm_bench.py > gpurun_out/gemm_bench.log 2>&1; echo "gemmbench rc=$?" ;;
    retest) timeout 900 python -m pytest tests/test_kernels_gpu.py tests/test_parity_gpu.py -m gpu -q --no-header -p no:cacheprovider -k "bf16_logits or vllm_fixture or preemption or abort" > gpurun_out/retest.log 2>&1; echo "retest rc=$?" ;;
    stl) TGIS_DEBUG_LAUNCH=1 TGIS_ENGINE_LIB=$PWD/vllm_tgis_adapter_b200/lib/libtgis_engine_stl.so timeout 300 python scripts/step_timeline.py 32 32 512 > gpurun_out/step_timeline_b32.log 2>&1; echo "stl rc=$?"; TGIS_DEBUG_LAUNCH=1 TGIS_ENGINE_LIB=$PWD/vllm_tgis_adapter_b200/lib/libtgis_engine_stl.so timeout 300 python scripts/step_timeline.py 32 64 512 > gpurun_out/step_timeline_b64.log 2>&1 ;;
    xcheck) timeout 1500 python scripts/vllm_crosscheck.py check > gpurun_out/xcheck.log 2>&1; echo "xcheck rc=$?" ;;
    xcheck_small) timeout 900 python scripts/vllm_crosscheck.py check --configs tiny > gpurun_out/xcheck.log 2>&1; echo "xcheck rc=$?" ;;
    vllmbench) timeout 1500 python scripts/vllm_crosscheck.py bench --batches 32 64 > gpurun_out/vllmbench.log 2>&1; echo "vllmbench rc=$?" ;;
    sampbench) timeout 300 python scripts/sampler_bench.py > gpurun_out/sampler_bench.log 2>&1; echo "sampbench rc=$?" ;;
    bench_cfg0) timeout 600 python bench.py --model 125m --batch 1 --cpu-layers 12 --steps 5 --warmup 3 > gpurun_out/bench_cfg0.log 2> gpurun_out/bench_cfg0.err; echo "bench_cfg0 rc=$?" ;;
    *) echo "unknown stage $st" ;;
  esac
done
tail -n 6 gpurun_out/*.log gpurun_out/*.err 2>/dev/null | cut -c1-1500
