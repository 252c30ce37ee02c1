"""Measure bucketing (``--bucketing s``) and heterogeneous data (``--dirichlet-alpha``) on one GPU and print one JSON line.

(a) ``kernels``: the new kernels alone on the ResNet-18 arena (11.2 M parameters), P = 7 and 15 slots, s = 2, CUDA events over
    --kernel-iters launches each: the plan kernel, bucket update mode 7 against plain and NNM-mixed mode 3, the bucket cc_dist
    + mode 8 chain against the plain cc_dist + mode 5 chain, and the bucket table + fold kernels.
(b) ``rate``: device-timed steps/s of the flagship job (``bench.py``'s configuration: ResNet-18 / CIFAR-10, batch 128, bf16,
    captured graph) at 15 workers, --worker-fail 3, s = 2: the median and centered clipping with and without bucketing, and
    Krum at --worker-fail 2, with the kernels launched per step and whether the PS pipelines.  Every arm runs in its own
    process; the arms alternate over --rate-rounds.
(c) ``loss``: final training loss after --steps steps, 15 workers, 3 liars, under IID data and --dirichlet-alpha 0.1 / 0.3,
    for baseline, bucketing (s = 2) and NNM, with the median, the geometric median and centered clipping (the last with the
    worker-momentum recipe; NNM has no centered clipping), under none / alie / minmax.  Single short runs on synthetic data.

    python tools/bench_bucketing.py [--parts kernels rate loss] [--out FILE]
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

RATE_ARMS = (("coordinate_median", 0, 3), ("coordinate_median", 2, 3), ("centered_clip", 0, 3), ("centered_clip", 2, 3),
             ("krum", 0, 2), ("krum", 2, 2))
ATTACKS = ("none", "alie", "minmax")
ALPHAS = (None, 0.1, 0.3)
RULES = ("coordinate_median", "geometric_median", "centered_clip")


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
    from draco_b200 import JobConfig
    from draco_b200.codes.bucketing import bucket_schedule
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    from draco_b200.parallel.ps import hyperparams_tensor
    dev = torch.device("cuda", 0)
    L = ArenaLayout.from_model(build_model("ResNet18", num_classes=10), bf16=True, channels_last=True)
    T, res = L.ntensors, []
    hp = hyperparams_tensor(JobConfig(lr=0.01, momentum=0.9), dev)
    params, mom = torch.zeros(L.total, device=dev), torch.zeros(L.total, device=dev)
    step = torch.ones(1, dtype=torch.int64, device=dev)
    cnt = torch.zeros(4, dtype=torch.int32, device=dev)
    upd = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1])
    for P in (7, 15):
        s, f = 2, 1 if P == 7 else 3
        nb = -(-P // s)
        slab = torch.randn(P, L.total, device=dev)
        sched = torch.from_numpy(bucket_schedule(P, 16, 1)).to(dev)
        masks = torch.zeros(nb, dtype=torch.int32, device=dev)
        scales = torch.zeros(nb, dtype=torch.float32, device=dev)
        K.wbucket_plan(sched, s, step_ptr=step, masks=masks, scales=scales)
        mix = torch.zeros(P, T, dtype=torch.int32, device=dev)
        pair = torch.zeros(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
        K.nnm_mix(L, slab, L.total, P, f, pair, mix, mixed_out=False)
        center = torch.zeros(L.total, device=dev)
        part_b = torch.zeros(L.ntiles, nb, dtype=torch.float64, device=dev)
        part_p = torch.zeros(L.ntiles, P, dtype=torch.float64, device=dev)
        w_b, w_p = torch.zeros(T, nb, device=dev), torch.zeros(T, P, device=dev)
        tab = torch.zeros(T, nb * (nb - 1) // 2, dtype=torch.float64, device=dev)
        sel = torch.ones(1, T, dtype=torch.int32, device=dev)
        wsel, wts = torch.zeros(s, T, dtype=torch.int32, device=dev), torch.zeros(T, s, device=dev)
        row = {"P": P, "s": s, "nb": nb, "slab_MB": round(P * L.total * 4 / 1e6, 1)}
        row["plan_us"] = _time(lambda: K.wbucket_plan(sched, s, step_ptr=step, masks=masks, scales=scales), iters)
        row["median_mode7_buckets_us"] = _time(lambda: K.wbucket_update(L, slab, L.total, masks=masks, scales=scales,
                                                                          trim=(nb - 1) // 2, **upd), iters)
        row["median_mode3_plain_us"] = _time(lambda: K.aggregate_update(L, slab, L.total, K=P, scale=1.0 / (P - 2 * ((P - 1) // 2)),
                                                                          trim=(P - 1) // 2, **upd), iters)
        row["median_mode3_nnm_mixed_us"] = _time(lambda: K.aggregate_update(
            L, slab, L.total, K=P, scale=1.0 / (P - 2 * ((P - 1) // 2)), trim=(P - 1) // 2, mix=mix, mix_f=f, **upd), iters)

        def cc_bucket():
            K.wbucket_cc_dist(L, slab, L.total, masks=masks, scales=scales, center=center, partials=part_b)
            K.centered_clip_weights(L, nb, 0.5, part_b, w_b)
            K.wbucket_cc_update(L, slab, L.total, masks=masks, scales=scales, center=center, weights=w_b, **upd)

        def cc_plain():
            K.centered_clip_dist(L, slab, L.total, P, center, part_p)
            K.centered_clip_weights(L, P, 0.5, part_p, w_p)
            K.centered_clip_update(L, slab, L.total, center=center, weights=w_p, K=P, **upd)
        row["cc_chain_buckets_us"] = _time(cc_bucket, iters)
        row["cc_chain_plain_us"] = _time(cc_plain, iters)
        row["table_us"] = _time(lambda: K.wbucket_table(L, P, masks=masks, raw_d2=pair, wb_d2=tab), iters)
        row["fold_krum_us"] = _time(lambda: K.wbucket_fold(L, P, masks=masks, weights=wts, select=sel, m=1, wsel=wsel), iters)
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
            mode, s, f = arm
            o = spawn(dict(kind="rate", approach="baseline", mode=mode, s=s, f=f, err_mode="rev_grad", steps=steps, warmup=warmup))
            if "error" in o:
                errors.append(o)
                continue
            runs[arm].append(round(o["steps_per_s"], 2))
            info[arm] = (o["kernels_per_step"], o["pipelined_ps"])
    res = []
    for (mode, s, f), v in runs.items():
        k, pipe = info.get((mode, s, f), (None, None))
        res.append({"mode": mode, "bucketing": s, "worker_fail": f, "steps_per_s": v, "median": statistics.median(v) if v else None,
                    "kernels_per_step": k, "pipelined_ps": pipe})
    return res + errors


def bench_loss(steps: int) -> list:
    res = []
    for alpha in ALPHAS:
        for err in ATTACKS:
            for rule in RULES:
                for row, approach, s in (("baseline", "baseline", 0), ("bucketing", "baseline", 2), ("nnm", "nnm", 0)):
                    if approach == "nnm" and rule == "centered_clip":
                        continue
                    res.append(spawn(dict(kind="loss", row=row, approach=approach, mode=rule, s=s, f=3, err_mode=err, alpha=alpha,
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
    ap.add_argument("--steps", type=int, default=35)
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
        out["loss"] = bench_loss(a.steps)
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
