#!/bin/bash
# Round-end benchmark sweep:  gpurun --gpus N -- bash tools/final_sweep.sh N [headline|extra|all] [steps]
#   headline : ResNet-18 / r=3 vote / 3 sign-flip adversaries, fused path and the NCCL reference-faithful baseline
#   extra    : the other configurations (VGG-11 cyclic, ResNet-18 geometric median / krum, ResNet-50 r=5) on the fused path
# Every run writes its JSON line to gpurun_out/sweep/<name>_N<N>.log; copy the ones to be judged into profiles/bench/.
cd "${GRAFT_REPO_ROOT:-$(dirname "$0")/..}"
N=${1:-1}; WHAT=${2:-all}; STEPS=${3:-60}
OUT=gpurun_out/sweep; mkdir -p $OUT
python -m draco_b200.build > $OUT/build_N$N.log 2>&1
PORT=29530
run() {  # name, bench args...
  local name=$1; shift
  PORT=$((PORT + 1))
  if [ "$N" = "1" ]; then
    timeout -k 10 420 python bench.py --gpus 1 --steps $STEPS --warmup 5 "$@" > $OUT/${name}_N$N.log 2>&1
  else
    timeout -k 10 420 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $PORT \
      bench.py --gpus $N --steps $STEPS --warmup 5 "$@" > $OUT/${name}_N$N.log 2>&1
  fi
  echo "$name N=$N rc=$? $(grep -o '"value": [0-9.e+-]*' $OUT/${name}_N$N.log | head -1) $(grep -o '"e2e": {"value": [0-9.e+-]*' $OUT/${name}_N$N.log | head -1)"
}
if [ "$WHAT" = "headline" ] || [ "$WHAT" = "all" ]; then
  run resnet18_vote_ours --impl ours
  run resnet18_vote_nccl --impl nccl
fi
if [ "$WHAT" = "extra" ] || [ "$WHAT" = "all" ]; then
  run vgg11_cyclic_s1_ours --impl ours --network VGG11 --approach cyclic --worker-fail 1 --err-mode random
  run resnet18_geomedian_ours --impl ours --approach baseline --mode geometric_median
  run resnet18_krum_ours --impl ours --approach baseline --mode krum
  run resnet50_vote_r5_ours --impl ours --network ResNet50 --group-size 5 --worker-fail 2 --batch-size 64
fi
if [ "$WHAT" = "extranccl" ]; then
  run vgg11_cyclic_s1_nccl --impl nccl --network VGG11 --approach cyclic --worker-fail 1 --err-mode random
  run resnet18_geomedian_nccl --impl nccl --approach baseline --mode geometric_median
fi
