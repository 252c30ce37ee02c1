#!/bin/bash
# round-2 measurement bundle (1 GPU): headline bench (ours / nccl_flat / ps-stream variant), failing-test recheck, small ncu captures
cd "${GRAFT_REPO_ROOT:-$(dirname "$0")/..}"
mkdir -p gpurun_out
python -m draco_b200.build > gpurun_out/env.log 2>&1
for s in "$@"; do
  case $s in
    alltests) timeout -k 10 1500 python -m pytest tests/ -q -m gpu -p no:cacheprovider -x > gpurun_out/t_all.log 2>&1; echo "alltests rc=$?"; tail -n 4 gpurun_out/t_all.log | cut -c1-300 ;;
    smoke) timeout -k 10 300 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/smoke.log 2>&1; echo "smoke rc=$?"; tail -n 3 gpurun_out/smoke.log ;;
    recheck) timeout -k 10 600 python -m pytest tests/test_fused_engine_gpu.py -q -m gpu -p no:cacheprovider -k "compress or phase_times or two_processes or dropout or library_op" > gpurun_out/t_recheck.log 2>&1; echo "recheck rc=$?" ;;
    gemmtests) timeout -k 10 600 python -m pytest tests/test_gemm_gpu.py -q -m gpu -p no:cacheprovider -k "gemm or linear" > gpurun_out/t_gemm.log 2>&1; echo "gemmtests rc=$?" ;;
    gemmbench) timeout -k 10 600 python tools/bench_gemm.py --json gpurun_out/gemm_bench.json > gpurun_out/gemm_bench.log 2>&1; echo "gemmbench rc=$?" ;;
    wgradstream) timeout -k 10 600 python -m pytest tests/test_fused_engine_gpu.py -q -m gpu -p no:cacheprovider -k "wgrad_side or two_processes" > gpurun_out/t_wgradstream.log 2>&1; echo "wgradstream rc=$?"
                 timeout -k 10 600 python tools/bench_worker.py > gpurun_out/bench_worker.log 2>&1; grep "ms per" gpurun_out/bench_worker.log ;;
    clustersweep) timeout -k 10 300 python -m pytest tests/test_gemm_gpu.py -q -m gpu -p no:cacheprovider -x -k "tap or convg or cluster or statistics or block_fusion" > gpurun_out/t_cluster.log 2>&1; echo "cluster tests rc=$?"; tail -n 5 gpurun_out/t_cluster.log
                 timeout -k 10 600 python tools/sweep_conv_cluster.py > gpurun_out/conv_cluster_sweep.log 2>&1; echo "sweep rc=$?"; tail -n 3 gpurun_out/conv_cluster_sweep.log | cut -c1-400 ;;
    convtimeline) timeout -k 10 300 python tools/prof_conv_timeline.py > gpurun_out/conv_timeline.log 2>&1; echo "convtimeline rc=$?"; tail -n 14 gpurun_out/conv_timeline.log | cut -c1-420 ;;
    convbench) timeout -k 10 600 python tools/bench_conv.py > gpurun_out/conv_bench.log 2>&1; echo "convbench rc=$?" ;;
    bench1) timeout -k 10 600 python bench.py --gpus 1 --steps 20 --warmup 5 > gpurun_out/bench1.log 2>&1; echo "bench1 rc=$?" ;;
    bench1_flat) timeout -k 10 600 python bench.py --gpus 1 --steps 20 --warmup 5 --impl nccl_flat > gpurun_out/bench1_flat.log 2>&1; echo "bench1_flat rc=$?" ;;
    bench1_ps) CUDA_DEVICE_MAX_CONNECTIONS=32 timeout -k 10 600 python bench.py --gpus 1 --steps 20 --warmup 5 --ps-stream > gpurun_out/bench1_psstream.log 2>&1; echo "bench1_ps rc=$?" ;;
    ncu_small) timeout -k 10 900 ncu --set full --clock-control none --import-source on -k regex:"convg_tcgen05|conv_halo|wgrad_halo|bn_bwd|bn_apply|stem_" -s 10 -c 14 -f -o gpurun_out/prof_conv python tools/prof_conv.py > gpurun_out/ncu_conv.log 2>&1; echo "ncu_small rc=$?" ;;
    launches) timeout -k 10 900 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/launches.csv python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/launches.log 2>&1; echo "launches rc=$?" ;;
  esac
done
tail -n 6 gpurun_out/t_recheck.log gpurun_out/t_gemm.log gpurun_out/gemm_bench.log gpurun_out/bench1*.log 2>/dev/null | cut -c1-1500
