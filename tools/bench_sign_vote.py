"""Measure signSGD with majority vote (``--mode sign_vote``) on one GPU and print one JSON line.

(a) ``kernels``: CUDA-event time per launch over --kernel-iters launches on the ResNet-18 arena (bf16 layout, arena-mode
    gradients, a local destination slot): the sign push against the plain and worker-momentum pushes, and update-kernel mode 6
    against mode 0 (the mean) at P = 7, 15 and 31 rows, SGD-momentum, no broadcast destination.  Each entry carries the bytes the
    algorithm needs (``bytes``) and their share of 3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth (``hbm_share``).
(b) ``step_rate``: device-timed steps/s of the flagship job (``bench.py``'s configuration: ResNet-18 / CIFAR-10, batch 128, bf16,
    captured graph) at 7 and 15 workers and ``--worker-fail 3`` under rev_grad: sign_vote against normal (the mean) and the
    pipelined coordinate-wise median, with the kernels launched per step.
(c) ``training``: final training loss after --steps steps, 15 workers, 3 liars, under none / rev_grad / constant: the Signum recipe
    (sign_vote, --worker-momentum 0.9 --momentum 0) against the coordinate-wise median (PS momentum 0.9, lr 0.01), over the --lrs
    grid for Signum.  Single short runs on synthetic data.

Every arm runs in its own process; the arms of (a) and (b) alternate over their rounds.

    python tools/bench_sign_vote.py [--parts kernels rate training] [--lrs 1e-4 1e-3] [--out FILE]
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

HBM_BYTES_PER_S = 3.35e12
KERNEL_ARMS = (("push", "plain"), ("push", "wmom"), ("push", "sign"), ("push", "sign_wmom"),
               *[(kind, P) for P in (7, 15, 31) for kind in ("update_mean", "update_sign")])
RATE_ARMS = [(P, mode) for P in (7, 15) for mode in ("sign_vote", "normal", "coordinate_median")]
ATTACKS = ("none", "rev_grad", "constant")


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


def kernel_one(spec: dict) -> dict:
    """One kernel arm: warm up, then CUDA events around ``iters`` launches."""
    import torch
    from draco_b200 import JobConfig
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    from draco_b200.parallel.ps import hyperparams_tensor
    dev = torch.device("cuda", 0)
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    D = L.total
    n16 = sum(s.numel for s in L.specs if s.is_bf16)
    n32 = sum(s.numel for s in L.specs if not s.is_bf16)
    step = torch.ones(1, dtype=torch.int64, device=dev)
    cnt = torch.zeros(4, dtype=torch.int32, device=dev)
    kind, arg = spec["kind"], spec["arg"]
    if kind == "push":
        g32 = torch.randn(D, device=dev)
        g16 = torch.randn(D, device=dev).to(torch.bfloat16)
        sign, wm = arg in ("sign", "sign_wmom"), arg in ("wmom", "sign_wmom")
        dst = torch.zeros(D // 32 if sign else D, dtype=torch.float32, device=dev)
        wmom = L.new_arena(dev) if wm else None
        # gradients read once (bf16 or fp32 per tensor), the slot written, the momentum state read and written
        nbytes = 2 * n16 + 4 * n32 + (D // 8 if sign else 4 * D) + (8 * D if wm else 0)

        def launch():
            K.push_encode(L, [g32], [g16], dst, step_ptr=step, worker=0, done_counter=cnt[0:1], wmom=wmom,
                          wm_beta=0.9 if wm else 0.0, sign=sign)
    else:
        P = int(arg)
        sign = kind == "update_sign"
        slab = (torch.randint(-2 ** 31, 2 ** 31 - 1, (P, D // 32), dtype=torch.int64, device=dev).to(torch.int32) if sign
                else torch.randn(P, D, device=dev) * 1e-3)
        params, mom = torch.randn(D, device=dev), torch.zeros(D, device=dev)
        hp = hyperparams_tensor(JobConfig(lr=1e-6, momentum=0.9), dev)
        kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1])
        # the P rows read, params and momentum read and written
        nbytes = (P * D // 8 if sign else 4 * P * D) + 16 * D

        def launch():
            if sign:
                K.sign_vote_update(L, slab, D // 32, P=P, **kw)
            else:
                K.aggregate_update(L, slab, D, K=P, scale=1.0 / P, **kw)
    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(spec["iters"]):
        launch()
    e.record()
    torch.cuda.synchronize()
    us = s.elapsed_time(e) * 1e3 / spec["iters"]
    return dict(spec, us=round(us, 2), bytes=nbytes, hbm_share=round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3))


def job_one(spec: dict) -> dict:
    import torch
    from draco_b200 import JobConfig
    from draco_b200.parallel.trainer import Trainer
    steps = spec["warmup"] + spec["steps"]
    cfg = JobConfig(network="ResNet18", dataset="Cifar10", approach="baseline", mode=spec["mode"], batch_size=128,
                    num_workers=spec["P"], worker_fail=3, err_mode=spec["err_mode"], lr=spec["lr"], momentum=spec["momentum"],
                    worker_momentum=spec["worker_momentum"], max_steps=steps + 8, eval_freq=10 ** 9, transport="nvl",
                    dtype="bf16", cuda_graphs=True, compress_grad="None", synthetic_size=8192, log_interval=10 ** 9)
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    out = dict(spec)
    if spec["kind"] == "rate":
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


def bench_kernels(rounds: int, iters: int) -> list:
    runs, errors, last = {arm: [] for arm in KERNEL_ARMS}, [], {}
    for r in range(rounds):
        for kind, arg in (KERNEL_ARMS if r % 2 == 0 else KERNEL_ARMS[::-1]):
            o = spawn(dict(kind=kind, arg=arg, iters=iters))
            if "error" in o:
                errors.append(o)
                continue
            runs[(kind, arg)].append(o["us"])
            last[(kind, arg)] = o
    res = []
    for arm, v in runs.items():
        if not v:
            continue
        us = statistics.median(v)
        nbytes = last[arm]["bytes"]
        res.append({"kernel": arm[0], "arg": arm[1], "us": v, "median_us": us, "bytes": nbytes,
                    "hbm_share": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)})
    return res + errors


def bench_rate(rounds: int, steps: int, warmup: int) -> list:
    runs = {arm: [] for arm in RATE_ARMS}
    info, errors = {}, []
    for r in range(rounds):
        for P, mode in (RATE_ARMS if r % 2 == 0 else RATE_ARMS[::-1]):
            sign = mode == "sign_vote"
            o = spawn(dict(kind="rate", mode=mode, P=P, err_mode="rev_grad", momentum=0.0 if sign else 0.9,
                           worker_momentum=0.9 if sign else 0.0, lr=1e-4 if sign else 0.01, steps=steps, warmup=warmup))
            if "error" in o:
                errors.append(o)
                continue
            runs[(P, mode)].append(round(o["steps_per_s"], 2))
            info[(P, mode)] = (o["kernels_per_step"], o["pipelined_ps"])
    res = []
    for (P, mode), v in runs.items():
        k, pipe = info.get((P, mode), (None, None))
        res.append({"workers": P, "mode": mode, "steps_per_s": v, "median": statistics.median(v) if v else None,
                    "kernels_per_step": k, "pipelined_ps": pipe})
    return res + errors


def bench_training(steps: int, lrs: list) -> list:
    res = []
    for err in ATTACKS:
        arms = [dict(mode="sign_vote", momentum=0.0, worker_momentum=0.9, lr=lr) for lr in lrs]
        arms.append(dict(mode="coordinate_median", momentum=0.9, worker_momentum=0.0, lr=0.01))
        for arm in arms:
            res.append(spawn(dict(kind="loss", P=15, err_mode=err, steps=steps, warmup=0, **arm)))
    return res


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--one", type=str, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--parts", nargs="+", default=["kernels", "rate", "training"], choices=("kernels", "rate", "training"))
    ap.add_argument("--kernel-rounds", type=int, default=2)
    ap.add_argument("--kernel-iters", type=int, default=200)
    ap.add_argument("--rate-rounds", type=int, default=2)
    ap.add_argument("--rate-steps", type=int, default=30)
    ap.add_argument("--rate-warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=35)
    ap.add_argument("--lrs", type=float, nargs="+", default=[1e-4, 1e-3])
    ap.add_argument("--out", type=str, default=None)
    a = ap.parse_args()
    if a.one is not None:
        spec = json.loads(a.one)
        print(json.dumps(kernel_one(spec) if spec["kind"].startswith(("push", "update")) else job_one(spec)), flush=True)
        return 0
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device visible"}), flush=True)
        return 1
    t0 = time.time()
    out = {"gpu": gpu_info(), "note": "training: single short runs on synthetic data"}
    if "kernels" in a.parts:
        out["kernels"] = bench_kernels(a.kernel_rounds, max(a.kernel_iters, 200))
    if "rate" in a.parts:
        out["step_rate"] = bench_rate(a.rate_rounds, a.rate_steps, a.rate_warmup)
    if "training" in a.parts:
        out["training"] = bench_training(a.steps, a.lrs)
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
