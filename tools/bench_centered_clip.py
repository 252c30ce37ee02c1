"""Measure centered clipping (``--mode centered_clip --clip-tau``) on one GPU and print one JSON line.

(a) ``step_rate``: device-timed steps/s of the flagship job (``bench.py``'s configuration: ResNet-18 / CIFAR-10, batch 128, bf16,
    captured graph) at 15 workers and ``--worker-fail 3`` under rev_grad, centered clipping against the pipelined coordinate-wise
    median and against multi-Krum, each under ``--approach baseline`` and ``--approach detox`` (groups of 3), with the kernels
    launched per step.  Every arm runs in its own process; the arms alternate over --rate-rounds.
(b) ``robustness``: final training loss after --steps steps, 15 workers, 3 liars, for centered clipping with PS momentum 0.9
    (lr 0.01) and with worker momentum 0.9 and no PS momentum at lr 0.1 (the same effective step, see the README's worker-momentum
    section), under none / alie / minmax, over the --taus grid.  Single short runs on synthetic data.

    python tools/bench_centered_clip.py [--parts rate robustness] [--taus 0.05 0.5] [--out FILE]
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

RATE_ARMS = (("baseline", "centered_clip"), ("baseline", "coordinate_median"), ("baseline", "multi_krum"),
             ("detox", "centered_clip"), ("detox", "coordinate_median"), ("detox", "multi_krum"))
ATTACKS = ("none", "alie", "minmax")
MOMENTA = {"ps_momentum": dict(momentum=0.9, worker_momentum=0.0, lr=0.01),
           "worker_momentum_lr10": dict(momentum=0.0, worker_momentum=0.9, lr=0.1)}


def gpu_info() -> dict:
    """Card name, power limit and max SM clock, read in the same call as the measurement."""
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except Exception as e:          # the measurement still stands; the card's limits are then unknown
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def run_one(spec: dict) -> dict:
    import torch
    from draco_b200 import JobConfig
    from draco_b200.parallel.trainer import Trainer
    steps = spec["warmup"] + spec["steps"]
    cfg = JobConfig(network="ResNet18", dataset="Cifar10", approach=spec["approach"], mode=spec["mode"], batch_size=128,
                    num_workers=15, group_size=3, worker_fail=3, err_mode=spec["err_mode"], lr=spec["lr"],
                    momentum=spec["momentum"], worker_momentum=spec["worker_momentum"], clip_tau=spec.get("tau"),
                    max_steps=steps + 8, eval_freq=10 ** 9, transport="nvl", dtype="bf16", cuda_graphs=True,
                    compress_grad="None", synthetic_size=8192, log_interval=10 ** 9)
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
        out["pipelined_ps"] = bool(t.engine.pipeline_ps)
    else:
        losses = []
        for _ in range(steps):
            m = t.train_step_pipelined()
            if m is not None:
                losses.append(m["loss"])
        losses.append(t.drain()["loss"])
        out["final_loss"] = losses[-1]
    t.close()
    return out


def spawn(spec: dict) -> dict:
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", json.dumps(spec)], capture_output=True, text=True,
                       cwd=ROOT, timeout=1800)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        return dict(spec, error=(r.stderr or r.stdout)[-1500:])
    return json.loads(lines[-1])


def bench_rate(rounds: int, steps: int, warmup: int, tau: float) -> list:
    runs = {arm: [] for arm in RATE_ARMS}
    info, errors = {}, []
    for r in range(rounds):
        for arm in (RATE_ARMS if r % 2 == 0 else RATE_ARMS[::-1]):
            approach, mode = arm
            o = spawn(dict(kind="rate", approach=approach, mode=mode, err_mode="rev_grad", momentum=0.9, worker_momentum=0.0,
                           lr=0.01, tau=tau if mode == "centered_clip" else None, steps=steps, warmup=warmup))
            if "error" in o:
                errors.append(o)
                continue
            runs[arm].append(round(o["steps_per_s"], 2))
            info[arm] = (o["kernels_per_step"], o["pipelined_ps"])
    res = []
    for (approach, mode), v in runs.items():
        k, pipe = info.get((approach, mode), (None, None))
        res.append({"approach": approach, "mode": mode, "steps_per_s": v, "median": statistics.median(v) if v else None,
                    "kernels_per_step": k, "pipelined_ps": pipe})
    return res + errors


def bench_robustness(steps: int, taus: list) -> list:
    res = []
    for err in ATTACKS:
        for tau in taus:
            for arm, mom in MOMENTA.items():
                o = spawn(dict(kind="loss", approach="baseline", mode="centered_clip", err_mode=err, tau=tau, steps=steps, warmup=0,
                               arm=arm, **mom))
                res.append(o)
    return res


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--one", type=str, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--parts", nargs="+", default=["rate", "robustness"], choices=("rate", "robustness"))
    ap.add_argument("--rate-rounds", type=int, default=2)
    ap.add_argument("--rate-steps", type=int, default=30)
    ap.add_argument("--rate-warmup", type=int, default=5)
    ap.add_argument("--rate-tau", type=float, default=0.05)
    ap.add_argument("--steps", type=int, default=35)
    ap.add_argument("--taus", type=float, nargs="+", default=[0.05, 0.5])
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
    out = {"gpu": gpu_info(), "note": "single short runs on synthetic data"}
    if "rate" in a.parts:
        out["step_rate"] = bench_rate(a.rate_rounds, a.rate_steps, a.rate_warmup, a.rate_tau)
    if "robustness" in a.parts:
        out["robustness"] = bench_robustness(a.steps, a.taus)
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
