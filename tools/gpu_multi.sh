#!/bin/bash
# multi-GPU measurement bundle: `gpurun --gpus N -- bash tools/gpu_multi.sh N stage...`   (logs under gpurun_out/multi_N<N>/)
cd "${GRAFT_REPO_ROOT:-$(dirname "$0")/..}"
N=$1; shift
OUT=gpurun_out/multi_N$N
mkdir -p $OUT
python -m draco_b200.build > $OUT/env.log 2>&1
nvidia-smi -L >> $OUT/env.log 2>&1
nvidia-smi topo -m >> $OUT/env.log 2>&1
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
for s in "$@"; do
  case $s in
    bench)      timeout -k 10 900 $TR --master-port 29611 bench.py --gpus $N --steps 30 --warmup 5 > $OUT/bench_ours.log 2> $OUT/bench_ours.err; echo "bench rc=$?" ;;
    timeline)   timeout -k 10 600 $TR --master-port 29615 bench.py --gpus $N --steps 10 --warmup 5 --skip-e2e --sanity-steps 0 --timeline $OUT/timeline $TIMELINE_ARGS > $OUT/timeline.log 2>&1; echo "timeline rc=$?" ;;
    timeline_e2e) timeout -k 10 600 $TR --master-port 29621 bench.py --gpus $N --steps 10 --warmup 5 --sanity-steps 0 --timeline-e2e $OUT/timeline_e2e $TIMELINE_ARGS > $OUT/timeline_e2e.log 2>&1; echo "timeline_e2e rc=$?" ;;
    bench_flat) timeout -k 10 900 $TR --master-port 29612 bench.py --gpus $N --steps 30 --warmup 5 --impl nccl_flat > $OUT/bench_flat.log 2> $OUT/bench_flat.err; echo "bench_flat rc=$?" ;;
    bench_nccl) timeout -k 10 900 $TR --master-port 29613 bench.py --gpus $N --steps 10 --warmup 3 --impl nccl > $OUT/bench_nccl.log 2> $OUT/bench_nccl.err; echo "bench_nccl rc=$?" ;;
    bench_wf1)  timeout -k 10 900 $TR --master-port 29614 bench.py --gpus $N --steps 30 --warmup 5 --worker-fail 1 --sanity-steps 0 > $OUT/bench_ours_wf1.log 2> $OUT/bench_ours_wf1.err; echo "bench_wf1 rc=$?" ;;
    sweep)      NCCL_DEBUG=WARN timeout -k 10 900 $TR --master-port 29615 tools/bench_push.py > $OUT/push_sweep.log 2> $OUT/push_sweep.err; cp gpurun_out/push_sweep_N$N.json $OUT/ 2>/dev/null; echo "sweep rc=$?" ;;
    tests)      timeout -k 10 2400 python -m pytest tests/test_fused_engine_gpu.py -q -m multigpu -p no:cacheprovider > $OUT/t_multigpu.log 2>&1; echo "tests rc=$?" ;;
    tests_quick) timeout -k 10 900 python -m pytest tests/test_fused_engine_gpu.py -q -m multigpu -p no:cacheprovider -k "peer_memory_matches or nvls" > $OUT/t_multigpu_quick.log 2>&1; echo "tests_quick rc=$?" ;;
    nvlink)     timeout -k 10 600 python tools/prof_nvlink.py > $OUT/nvlink_timing.log 2>&1; echo "nvlink timing rc=$?"
                timeout -k 10 900 ncu --clock-control none --metrics gpu__time_duration.sum,nvltx__bytes.sum,nvlrx__bytes.sum,dram__bytes_read.sum,dram__bytes_write.sum,lts__t_bytes.sum -k regex:"push_encode|aggregate_update" -s 12 -c 6 --csv --log-file $OUT/nvlink_counters.csv python tools/prof_nvlink.py > $OUT/nvlink_ncu.log 2>&1; echo "nvlink ncu rc=$?" ;;
    sweep132)   PUSH_CTAS=132 timeout -k 10 900 $TR --master-port 29620 tools/bench_push.py > $OUT/push_sweep_132cta.log 2> $OUT/push_sweep_132cta.err; echo "sweep132 rc=$?" ;;
    test_equiv) timeout -k 10 1500 python -m pytest tests/test_fused_engine_gpu.py -q -m multigpu -p no:cacheprovider -k "equals_nccl" > $OUT/t_multigpu_equiv.log 2>&1; echo "test_equiv rc=$?" ;;
    geomed)     timeout -k 10 900 $TR --master-port 29616 bench.py --gpus $N --steps 30 --warmup 5 --approach baseline --mode geometric_median --sanity-steps 0 > $OUT/bench_geomed.log 2> $OUT/bench_geomed.err; echo "geomed rc=$?" ;;
    vgg_cyclic) timeout -k 10 900 $TR --master-port 29617 bench.py --gpus $N --steps 30 --warmup 5 --network VGG11 --approach cyclic --worker-fail 1 --err-mode constant --sanity-steps 0 > $OUT/bench_vgg_cyclic.log 2> $OUT/bench_vgg_cyclic.err; echo "vgg_cyclic rc=$?" ;;
    r50)        timeout -k 10 900 $TR --master-port 29618 bench.py --gpus $N --steps 20 --warmup 5 --network ResNet50 --group-size 5 --worker-fail 2 --batch-size 64 --sanity-steps 0 > $OUT/bench_resnet50.log 2> $OUT/bench_resnet50.err; echo "r50 rc=$?" ;;
    r50_imagenet) timeout -k 10 1200 $TR --master-port 29619 bench.py --gpus $N --steps 10 --warmup 3 --network ResNet50 --dataset ImageNet --group-size 5 --worker-fail 2 --batch-size 32 --sanity-steps 0 > $OUT/bench_resnet50_imagenet.log 2> $OUT/bench_resnet50_imagenet.err; echo "r50_imagenet rc=$?" ;;
  esac
done
tail -n 4 $OUT/*.log 2>/dev/null | cut -c1-900 | tail -n 60
tail -n 5 $OUT/*.err 2>/dev/null | cut -c1-300 | tail -n 30
