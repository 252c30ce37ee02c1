"""Time the fused PS update kernel alone (csrc/cuda/aggregate_update.cu): mode 0, the mean of P gradient rows, against mode 3,
the coordinate-wise trimmed mean and median, on the ResNet-18 (CIFAR) parameter arena.

Each call reads the P x D fp32 gradient slab once and reads + writes the fp32 parameters and momentum (SGD-momentum, no
broadcast destinations).  Timed with CUDA events over --iters back-to-back launches; the rules alternate over --rounds and the
median round is reported.  Bandwidth is the slab bytes (P * D * 4) per microsecond, also as a share of the H100 SXM data-sheet
HBM3 bandwidth of 3.35 TB/s (3.35e6 bytes/us); ``total_bytes_per_us`` adds the 16 * D bytes of parameter / momentum traffic.

    python tools/bench_aggregate.py [--workers 7 16] [--iters 200] [--rounds 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_US = 3.35e6


def gpu_info() -> dict:
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except Exception as e:          # the measurement still stands; the card's limits are then unknown
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workers", type=int, nargs="+", default=[7, 16])
    ap.add_argument("--trim", type=int, default=2, help="values dropped at each end by the trimmed mean (= --worker-fail)")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", type=str, default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device visible"}))
        return 1
    from draco_b200 import JobConfig
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    from draco_b200.parallel.ps import hyperparams_tensor

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    D = L.total
    hp = hyperparams_tensor(JobConfig(lr=0.01, momentum=0.9), dev)
    params = torch.zeros(D, device=dev)
    mom = torch.zeros(D, device=dev)
    step = torch.full((1,), 2, dtype=torch.int64, device=dev)
    cnt = torch.zeros(4, dtype=torch.int32, device=dev)
    lines = [dict(gpu_info(), arena="ResNet18/Cifar10", D=D, iters=a.iters, rounds=a.rounds)]
    for P in a.workers:
        slab = torch.randn(P, D, device=dev) * 1e-3
        rules = {"mean": dict(K=P, scale=1.0 / P),
                 f"trimmed_mean_b{a.trim}": dict(K=P, scale=1.0 / (P - 2 * a.trim), trim=a.trim),
                 "median": dict(K=P, scale=1.0 / (P - 2 * ((P - 1) // 2)), trim=(P - 1) // 2)}

        def launch(kw):
            K.aggregate_update(L, slab, D, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], **kw)

        for kw in rules.values():                                  # load the module, settle the clocks
            for _ in range(20):
                launch(kw)
        torch.cuda.synchronize()
        times = {name: [] for name in rules}
        for _ in range(a.rounds):
            for name, kw in rules.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.iters):
                    launch(kw)
                e.record()
                e.synchronize()
                times[name].append(s.elapsed_time(e) * 1e3 / a.iters)
        slab_bytes = P * D * 4
        for name, ts in times.items():
            us = sorted(ts)[len(ts) // 2]
            lines.append({"P": P, "rule": name, "mode": 0 if name == "mean" else 3, "us_per_call": round(us, 2),
                          "us_rounds": [round(t, 2) for t in ts], "slab_bytes": slab_bytes,
                          "slab_bytes_per_us": round(slab_bytes / us), "slab_share_of_3.35TBps": round(slab_bytes / us / HBM_BYTES_PER_US, 3),
                          "total_bytes_per_us": round((slab_bytes + 16 * D) / us)})
        del slab
    for ln in lines:
        print(json.dumps(ln), flush=True)
    if a.out:
        with open(a.out, "a") as fh:
            for ln in lines:
                fh.write(json.dumps(ln) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
