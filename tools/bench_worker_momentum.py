"""Measure worker-side momentum (``--worker-momentum``) on one GPU and print one JSON line.

(a) ``push``: the push kernel alone (csrc/cuda/push_encode.cu) on the ResNet-18 (CIFAR, bf16) arena, plain against the momentum
    build, into a local slot.  CUDA events over --iters back-to-back launches, the two builds alternated over --rounds, the
    median round reported.  ``bytes`` is the HBM traffic the algorithm needs: plain reads the gradient (2 B per bf16 element,
    4 B per fp32 one) and writes the fp32 slot; momentum adds the fp32 state read and written (8 B per element).
(b) ``step_rate``: device-timed steps/s of the flagship job (``bench.py``'s configuration) with beta = 0.9 against beta = 0, at
    the headline setting (7 workers, groups of 3) and at the robustness setting (15 workers, groups of 3, 3 liars), the arms
    alternated over --rate-rounds.  Each run is its own process.
(c) ``robustness``: final training loss of the robustness matrix.  Arms (--arms): PS momentum 0.9 with beta = 0, PS momentum 0
    with beta = 0.9, and the same at a 10x learning rate (the dampened state moves the parameters by lr * g at steady state, PS
    momentum 0.9 by 10 lr * g).  Rules: baseline coordinate_median / multi_krum / bulyan and nnm coordinate_median, 15 workers, 3 liars;
    attacks: none / alie / minmax.  --short-steps (35: the README tables' 5 warm-up + 30 timed steps) for every cell, and
    --long-steps for the cells listed in --long-cells.

    python tools/bench_worker_momentum.py [--parts push rate robustness] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RULES = (("baseline", "coordinate_median"), ("baseline", "multi_krum"), ("baseline", "bulyan"), ("nnm", "coordinate_median"))
ATTACKS = ("none", "alie", "minmax")
# dampened worker momentum moves the parameters by lr * g at steady state, PS momentum 0.9 by 10 lr * g: the third arm gives
# worker momentum the same effective step
ARMS = {"ps_momentum": dict(momentum=0.9, worker_momentum=0.0, lr=0.01),
        "worker_momentum": dict(momentum=0.0, worker_momentum=0.9, lr=0.01),
        "worker_momentum_lr10": dict(momentum=0.0, worker_momentum=0.9, lr=0.1)}


def gpu_info() -> dict:
    """Card name and power limit, read in the same call as the measurement."""
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except Exception as e:          # the measurement still stands; the card's limits are then unknown
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


# ------------------------------------------------------------------------------------------------ (a) the kernel alone
def bench_push(iters: int, rounds: int) -> dict:
    import torch
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    dev = torch.device("cuda", 0)
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    g32, g16 = L.new_arena(dev), L.new_arena(dev, torch.bfloat16)
    g = torch.Generator().manual_seed(0)
    for s in L.specs:
        v = torch.randn(s.numel, generator=g).to(dev) * 1e-2
        (g16 if s.is_bf16 else g32)[s.offset: s.offset + s.numel] = v.to(g16.dtype if s.is_bf16 else g32.dtype)
    slot, wm = L.new_arena(dev), L.new_arena(dev)
    step = torch.ones(1, dtype=torch.int64, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    grad_bytes = sum(s.numel * (2 if s.is_bf16 else 4) for s in L.specs)
    bytes_plain = grad_bytes + 4 * L.total
    bytes_wm = bytes_plain + 8 * L.total

    def launch(momentum: bool):
        K.push_encode(L, [g32], [g16], slot, step_ptr=step, worker=0, done_counter=cnt,
                      **(dict(wmom=wm, wm_beta=0.9) if momentum else {}))

    times = {False: [], True: []}
    for momentum in (False, True):                           # warm-up (module load, clocks)
        for _ in range(20):
            launch(momentum)
    torch.cuda.synchronize()
    for _ in range(rounds):
        for momentum in (False, True):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                launch(momentum)
            e.record()
            torch.cuda.synchronize()
            times[momentum].append(s.elapsed_time(e) * 1e3 / iters)
    out = {"arena_elements": L.total, "iters": iters, "rounds": rounds}
    for momentum, nbytes in ((False, bytes_plain), (True, bytes_wm)):
        us = statistics.median(times[momentum])
        out["momentum" if momentum else "plain"] = {"us": us, "bytes": nbytes, "bytes_per_us": nbytes / us,
                                                   "rounds_us": times[momentum]}
    out["momentum_over_plain"] = out["momentum"]["us"] / out["plain"]["us"]
    return out


# ------------------------------------------------------------------------------------------------ one job (own process)
def job_config(num_workers: int, worker_fail: int, approach: str, mode: str, err_mode: str, momentum: float,
               worker_momentum: float, steps: int, lr: float = 0.01):
    """bench.py's JobConfig for the flagship job, with the given rule, attack and momenta."""
    from draco_b200 import JobConfig
    return JobConfig(network="ResNet18", dataset="Cifar10", approach=approach, mode=mode, batch_size=128,
                     num_workers=num_workers, group_size=3, worker_fail=worker_fail, err_mode=err_mode, lr=lr, momentum=momentum,
                     worker_momentum=worker_momentum, max_steps=steps + 8, eval_freq=10 ** 9, transport="nvl", dtype="bf16",
                     cuda_graphs=True, compress_grad="None", synthetic_size=8192, log_interval=10 ** 9)


def run_one(spec: dict) -> dict:
    import torch
    from draco_b200.parallel.trainer import Trainer
    cfg = job_config(spec["num_workers"], spec["worker_fail"], spec["approach"], spec["mode"], spec["err_mode"], spec["momentum"],
                     spec["worker_momentum"], spec["warmup"] + spec["steps"], spec.get("lr", 0.01))
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    out = dict(spec)
    if spec["kind"] == "rate":
        cfg.data_on_device = True
        for _ in range(spec["warmup"]):
            t.train_step_async()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(spec["steps"]):
            t.train_step_async()
        e.record()
        torch.cuda.synchronize()
        out["steps_per_s"] = spec["steps"] / (s.elapsed_time(e) / 1e3)
        out["kernels_per_step"] = t.engine.kernels_per_step
    else:
        losses = []
        for _ in range(spec["warmup"] + spec["steps"]):
            m = t.train_step_pipelined()
            if m is not None:
                losses.append(m["loss"])
        losses.append(t.drain()["loss"])
        out["final_loss"] = losses[-1]
        out["loss_at"] = {str(k): losses[k - 1] for k in (10, 35, 100, 200) if k <= len(losses)}
    t.close()
    return out


def spawn(spec: dict) -> dict:
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", json.dumps(spec)], capture_output=True, text=True,
                       cwd=ROOT, timeout=1800)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        return dict(spec, error=(r.stderr or r.stdout)[-1500:])
    return json.loads(lines[-1])


def bench_rate(rounds: int, steps: int, warmup: int) -> list:
    settings = (("headline", 7, 3, "maj_vote", "maj_vote", "rev_grad"), ("robustness", 15, 3, "baseline", "coordinate_median", "rev_grad"))
    res = []
    for name, P, f, approach, mode, err in settings:
        runs = {0.0: [], 0.9: []}
        kps = {}
        for r in range(rounds):
            order = (0.0, 0.9) if r % 2 == 0 else (0.9, 0.0)
            for beta in order:
                o = spawn(dict(kind="rate", num_workers=P, worker_fail=f, approach=approach, mode=mode, err_mode=err, momentum=0.9,
                               worker_momentum=beta, steps=steps, warmup=warmup))
                if "error" in o:
                    res.append(o)
                    continue
                runs[beta].append(o["steps_per_s"])
                kps[beta] = o["kernels_per_step"]
        med = {b: statistics.median(v) if v else None for b, v in runs.items()}
        res.append({"setting": name, "num_workers": P, "worker_fail": f, "approach": approach, "mode": mode, "err_mode": err,
                    "steps_per_s_beta0": runs[0.0], "steps_per_s_beta0.9": runs[0.9], "kernels_per_step": kps,
                    "cost_pct": (100.0 * (1 - med[0.9] / med[0.0])) if med[0.0] and med[0.9] else None})
    return res


def bench_robustness(short: int, long: int, long_cells: list, arms: list, rules: list) -> list:
    res = []
    for approach, mode in (r for r in RULES if f"{r[0]}/{r[1]}" in rules):
        for err in ATTACKS:
            for arm, mom in ((k, v) for k, v in ARMS.items() if k in arms):     # arms alternate inside every cell
                steps = ([short] if short > 0 else []) + ([long] if f"{approach}/{mode}/{err}" in long_cells else [])
                for n in steps:
                    o = spawn(dict(kind="loss", num_workers=15, worker_fail=3, approach=approach, mode=mode, err_mode=err,
                                   steps=n, warmup=0, arm=arm, **mom))
                    res.append(o)
    return res


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--one", type=str, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--parts", nargs="+", default=["push", "rate", "robustness"], choices=("push", "rate", "robustness"))
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rate-rounds", type=int, default=2)
    ap.add_argument("--rate-steps", type=int, default=30)
    ap.add_argument("--rate-warmup", type=int, default=5)
    ap.add_argument("--short-steps", type=int, default=35)
    ap.add_argument("--long-steps", type=int, default=200)
    ap.add_argument("--long-cells", nargs="*", default=["baseline/coordinate_median/none", "baseline/coordinate_median/alie",
                                                         "baseline/multi_krum/none", "baseline/multi_krum/alie"])
    ap.add_argument("--arms", nargs="+", default=list(ARMS), choices=list(ARMS))
    ap.add_argument("--rules", nargs="+", default=[f"{a}/{m}" for a, m in RULES])
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if a.one is not None:
        print(json.dumps(run_one(json.loads(a.one))), flush=True)
        return 0
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device visible"}), flush=True)
        return 1
    t0 = time.time()
    out = {"gpu": gpu_info()}
    if "push" in a.parts:
        out["push"] = bench_push(a.iters, a.rounds)
    if "rate" in a.parts:
        out["step_rate"] = bench_rate(a.rate_rounds, a.rate_steps, a.rate_warmup)
    if "robustness" in a.parts:
        out["robustness"] = bench_robustness(a.short_steps, a.long_steps, a.long_cells, a.arms, a.rules)
    out["wall_s"] = time.time() - t0
    line = json.dumps(out)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    print(line, flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
