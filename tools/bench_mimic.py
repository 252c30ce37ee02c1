"""Measure the mimic and IPM attacks (``--err-mode mimic | ipm``) on one GPU and print one JSON line.

(a) ``kernels``: the attack kernels alone on the ResNet-18 arena (11.2 M parameters), P = 7 and 15 slots, CUDA events over
    --kernel-iters launches each: the six-kernel mimic chain in a warm-up step and after it, the IPM kernel and ALIE's kernel,
    with the bytes each needs (every honest slot read once, the liar slots written once; mimic's warm-up also reads and writes
    m, reads z, writes u, reads u and writes z) as a share of the H100 SXM's 3.35 TB/s.
(b) ``rate``: device-timed steps/s of the flagship job (``bench.py``'s configuration: ResNet-18 / CIFAR-10, batch 128, bf16,
    captured graph) at 15 workers, --worker-fail 3: alie, ipm and mimic under the median and centered clipping, with and
    without --bucketing 2, with the kernels launched per step and whether the PS pipelines.  Every arm runs in its own
    process; the arms alternate over --rate-rounds.
(c) ``loss``: final training loss after --steps steps (past mimic's default warm-up of 20 steps), 15 workers, 3 liars, under
    IID data and --dirichlet-alpha 0.1, for none / alie / ipm / mimic against the median (baseline, --bucketing 2, NNM) and
    centered clipping with the worker-momentum recipe (with and without --bucketing 2).  Single short runs on synthetic data.

    python tools/bench_mimic.py [--parts kernels rate loss] [--out FILE]
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

RATE_ARMS = tuple((err, mode, s) for mode in ("coordinate_median", "centered_clip") for s in (0, 2)
                  for err in ("alie", "ipm", "mimic"))
ATTACKS = ("none", "alie", "ipm", "mimic")
ALPHAS = (None, 0.1)
# (row, approach, mode, bucketing)
LOSS_ARMS = (("baseline", "baseline", "coordinate_median", 0), ("bucketing", "baseline", "coordinate_median", 2),
             ("nnm", "nnm", "coordinate_median", 0), ("cc", "baseline", "centered_clip", 0),
             ("cc_bucketing", "baseline", "centered_clip", 2))
HBM_TBPS = 3.35


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


def _time(fn, iters: int) -> float:
    """Median over 3 rounds of the mean device time of ``fn`` in microseconds (CUDA events around ``iters`` launches)."""
    import torch
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(3):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e) * 1e3 / iters)
    return round(statistics.median(out), 2)


def bench_kernels(iters: int) -> list:
    import torch
    from draco_b200.codes import adversary as A
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    dev = torch.device("cuda", 0)
    L = ArenaLayout.from_model(build_model("ResNet18", num_classes=10), bf16=True, channels_last=True)
    z0 = torch.from_numpy(A.mimic_z0([(s.offset, s.numel) for s in L.specs], L.total))
    D, res = L.num_params, []
    for P in (7, 15):
        f = 1 if P == 7 else 3
        n = P - f
        slab = torch.randn(P, L.total, device=dev)
        bm = torch.tensor([(1 << f) - 1], dtype=torch.int32, device=dev)          # slots 0 .. f-1 lie
        warm, after = (torch.ones(1, dtype=torch.int64, device=dev), torch.full((1,), 10 ** 6, dtype=torch.int64, device=dev))
        st = K.MimicState(L, P, dev, z0)
        att = dict(adv_bitmap=bm, adv_len=1)
        row = {"P": P, "liars": f, "slab_MB": round(P * L.total * 4 / 1e6, 1)}
        t = {
            "mimic_warmup_us": _time(lambda: K.mimic_step(L, slab, L.total, P, step_ptr=warm, warmup=10 ** 9, st=st, **att), iters),
            "mimic_after_us": _time(lambda: K.mimic_step(L, slab, L.total, P, step_ptr=after, warmup=1, st=st, **att), iters),
            "ipm_us": _time(lambda: K.ps_attack(L, slab, L.total, P, A.ATTACK_IPM, step_ptr=warm, z=0.1, **att), iters),
            "alie_us": _time(lambda: K.ps_attack(L, slab, L.total, P, A.ATTACK_ALIE, step_ptr=warm, z=1.0, **att), iters),
        }
        # bytes the algorithm needs: honest slots read once, liar slots written once (fp32); mimic after the warm-up reads z and
        # the honest slots for the projections, then x_k and writes the liars; in warm-up it also reads and writes m, reads the
        # honest slots, m and z again for u, writes and re-reads u (fp64) and writes z
        need = {"ipm_us": 4 * D * (n + f), "alie_us": 4 * D * (n + f),
                "mimic_after_us": 4 * D * (n + 1 + 1 + f),
                "mimic_warmup_us": 4 * D * (n + 1 + 2 + 1 + f) + 4 * D * (n + 2) + 8 * D * 2 + 4 * D}
        for k, us in t.items():
            row[k] = us
            row[k.replace("_us", "_MB")] = round(need[k] / 1e6, 1)
            row[k.replace("_us", "_hbm_share")] = round(need[k] / (us * 1e-6) / (HBM_TBPS * 1e12), 3)
        res.append(row)
    return res


def run_one(spec: dict) -> dict:
    import torch
    from draco_b200 import JobConfig
    from draco_b200.parallel.trainer import Trainer
    steps = spec["warmup"] + spec["steps"]
    cc = spec["mode"] == "centered_clip"
    cfg = JobConfig(network="ResNet18", dataset="Cifar10", approach=spec["approach"], mode=spec["mode"], batch_size=128,
                    num_workers=15, worker_fail=spec["f"], err_mode=spec["err_mode"], bucketing=spec["s"],
                    dirichlet_alpha=spec.get("alpha"), lr=0.1 if cc else 0.01, momentum=0.0 if cc else 0.9,
                    worker_momentum=0.9 if cc else 0.0, clip_tau=0.5 if cc else None, max_steps=steps + 8, eval_freq=10 ** 9,
                    transport="nvl", dtype="bf16", cuda_graphs=True, compress_grad="None", synthetic_size=8192,
                    log_interval=10 ** 9)
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


def bench_rate(rounds: int, steps: int, warmup: int) -> list:
    runs = {arm: [] for arm in RATE_ARMS}
    info, errors = {}, []
    for r in range(rounds):
        for arm in (RATE_ARMS if r % 2 == 0 else RATE_ARMS[::-1]):
            err, mode, s = arm
            o = spawn(dict(kind="rate", approach="baseline", mode=mode, s=s, f=3, err_mode=err, steps=steps, warmup=warmup))
            if "error" in o:
                errors.append(o)
                continue
            runs[arm].append(round(o["steps_per_s"], 2))
            info[arm] = (o["kernels_per_step"], o["pipelined_ps"])
    res = []
    for (err, mode, s), v in runs.items():
        k, pipe = info.get((err, mode, s), (None, None))
        res.append({"err_mode": err, "mode": mode, "bucketing": s, "steps_per_s": v, "median": statistics.median(v) if v else None,
                    "kernels_per_step": k, "pipelined_ps": pipe})
    return res + errors


def bench_loss(steps: int, attacks, alphas) -> list:
    res = []
    for alpha in alphas:
        for err in attacks:
            for row, approach, mode, s in LOSS_ARMS:
                res.append(spawn(dict(kind="loss", row=row, approach=approach, mode=mode, s=s, f=3, err_mode=err, alpha=alpha,
                                      steps=steps, warmup=0)))
    return res


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--one", type=str, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--parts", nargs="+", default=["kernels", "rate", "loss"], choices=("kernels", "rate", "loss"))
    ap.add_argument("--kernel-iters", type=int, default=100)
    ap.add_argument("--rate-rounds", type=int, default=2)
    ap.add_argument("--rate-steps", type=int, default=30)
    ap.add_argument("--rate-warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--loss-attacks", nargs="+", default=list(ATTACKS), choices=ATTACKS)
    ap.add_argument("--loss-alphas", nargs="+", type=float, default=[0.0, 0.1], help="0 = IID")
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
    if "kernels" in a.parts:
        out["kernels"] = bench_kernels(a.kernel_iters)
    if "rate" in a.parts:
        out["step_rate"] = bench_rate(a.rate_rounds, a.rate_steps, a.rate_warmup)
    if "loss" in a.parts:
        out["loss"] = bench_loss(a.steps, a.loss_attacks, [x or None for x in a.loss_alphas])
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
