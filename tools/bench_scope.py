"""Measure whole-model scope (``--rule-scope model``, ``--attack-scope model``) on one GPU and print one JSON line.

(a) ``kernels``: CUDA-event times of the new kernels alone on the ResNet-18 arena at P = 7 and 15 -- the pair-table scope fold,
    centered clipping's fold + model weights, and min-max's fold + model solve -- with the per-tensor kernels they replace.
(b) ``step_rate``: device-timed steps/s of the flagship job (``bench.py``'s configuration: ResNet-18 / CIFAR-10, batch 128, bf16,
    captured graph) at 15 workers and ``--worker-fail 3`` under rev_grad, tensor against model scope, for multi_krum, bulyan,
    nnm/coordinate_median and centered_clip under baseline and multi_krum under detox (groups of 3).  Every arm runs in its own
    process; the arms alternate over --rate-rounds.
(c) ``robustness``: final training loss after --steps steps, 15 workers, 3 liars, under none / alie / minmax, in both rule
    scopes and (for min-max) both attack scopes.  Centered clipping's tau grid is per scope: the whole-model norm is about
    sqrt(T) times one tensor's, so the model-scope grid is the tensor grid times sqrt(62) ~ 8 for ResNet-18.  Single short runs
    on synthetic data.

    python tools/bench_scope.py [--parts kernels rate robustness] [--out FILE]
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

from tools.bench_centered_clip import gpu_info  # noqa: E402

RATE_ARMS = (("baseline", "multi_krum"), ("baseline", "bulyan"), ("nnm", "coordinate_median"), ("baseline", "centered_clip"),
             ("detox", "multi_krum"))
ROBUST_ARMS = (("baseline", "multi_krum"), ("baseline", "bulyan"), ("nnm", "coordinate_median"), ("baseline", "centered_clip"))
ATTACKS = ("none", "alie", "minmax")
TAU = {"tensor": 0.05, "model": 0.4}                 # centered clipping: 0.05 per tensor, ~ sqrt(62) times that for the model


def bench_kernels(reps: int) -> list:
    import torch
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    dev = torch.device("cuda", 0)
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    T, res = L.ntensors, []

    def timed(name, P, fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        res.append({"kernel": name, "P": P, "us": round(s.elapsed_time(e) * 1e3 / reps, 2)})

    for P in (7, 15):
        g = torch.Generator().manual_seed(P)
        X = (torch.randn(P, L.total, generator=g) * torch.rand(P, 1, generator=g)).to(dev)
        pair = torch.rand(T, P * (P - 1) // 2, dtype=torch.float64, device=dev)
        timed("pair_scope_fold", P, lambda: K.pair_scope_fold(L, P, pair))
        v = torch.zeros(L.total, device=dev)
        partials = torch.zeros(L.ntiles, P, dtype=torch.float64, device=dev)
        K.centered_clip_dist(L, X, L.total, P, v, partials)
        dist = torch.zeros(T, P, dtype=torch.float64, device=dev)
        w = torch.zeros(T, P, dtype=torch.float32, device=dev)
        timed("cc_fold+cc_model_weights", P, lambda: K.centered_clip_model_weights(L, P, 1.0, partials, dist, w))
        timed("cc_weights (per tensor)", P, lambda: K.centered_clip_weights(L, P, 1.0, partials, w))
        ws = K.AttackWorkspace(L, P, dev)
        fold = K.attack_fold_buffer(L, P, dev)
        bitmap = torch.tensor([0b101], dtype=torch.int32, device=dev)
        step = torch.zeros(1, dtype=torch.int64, device=dev)
        K.ps_attack_model(L, X.clone(), L.total, P, adv_bitmap=bitmap, adv_len=1, step_ptr=step, ws=ws, fold=fold)
        a, _ = K._attack_args(L, X, L.total, P, 6, bitmap, 1, step, 0.0, ws, None, None)
        a.fold = fold.data_ptr()
        import ctypes as C
        lib = K.N.cuda()
        timed("attack_fold+attack_solve_model", P, lambda: lib.drc_attack_solve_model(C.byref(a), K._stream()))
        timed("attack_solve (per tensor)", P, lambda: lib.drc_attack_solve(C.byref(a), K._stream()))
    return res


def run_one(spec: dict) -> dict:
    import torch
    from draco_b200 import JobConfig
    from draco_b200.parallel.trainer import Trainer
    steps = spec["warmup"] + spec["steps"]
    cc = spec["mode"] == "centered_clip"
    cfg = JobConfig(network="ResNet18", dataset="Cifar10", approach=spec["approach"], mode=spec["mode"], batch_size=128,
                    num_workers=15, group_size=3, worker_fail=3, err_mode=spec["err_mode"], lr=0.01, momentum=0.9,
                    clip_tau=TAU[spec["rule_scope"]] if cc else None, rule_scope=spec["rule_scope"],
                    attack_scope=spec["attack_scope"], max_steps=steps + 8, eval_freq=10 ** 9, transport="nvl", dtype="bf16",
                    cuda_graphs=True, compress_grad="None", synthetic_size=8192, log_interval=10 ** 9)
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


def bench_rate(rounds: int, steps: int, warmup: int) -> list:
    arms = [(a, m, s) for a, m in RATE_ARMS for s in ("tensor", "model")]
    runs = {arm: [] for arm in arms}
    info, errors = {}, []
    for r in range(rounds):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            approach, mode, scope = arm
            o = spawn(dict(kind="rate", approach=approach, mode=mode, err_mode="rev_grad", rule_scope=scope, attack_scope="tensor",
                           steps=steps, warmup=warmup))
            if "error" in o:
                errors.append(o)
                continue
            runs[arm].append(round(o["steps_per_s"], 2))
            info[arm] = (o["kernels_per_step"], o["pipelined_ps"])
    res = []
    for arm, v in runs.items():
        k, pipe = info.get(arm, (None, None))
        res.append({"approach": arm[0], "mode": arm[1], "rule_scope": arm[2], "steps_per_s": v,
                    "median": statistics.median(v) if v else None, "kernels_per_step": k, "pipelined_ps": pipe})
    return res + errors


def bench_robustness(steps: int) -> list:
    res = []
    for approach, mode in ROBUST_ARMS:
        for err in ATTACKS:
            for rule_scope in ("tensor", "model"):
                for attack_scope in (("tensor", "model") if err == "minmax" else ("tensor",)):
                    res.append(spawn(dict(kind="loss", approach=approach, mode=mode, err_mode=err, rule_scope=rule_scope,
                                          attack_scope=attack_scope, steps=steps, warmup=0)))
    return res


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--one", type=str, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--parts", nargs="+", default=["kernels", "rate", "robustness"], choices=("kernels", "rate", "robustness"))
    ap.add_argument("--kernel-reps", type=int, default=200)
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
        out["kernels"] = bench_kernels(a.kernel_reps)
    if "rate" in a.parts:
        out["step_rate"] = bench_rate(a.rate_rounds, a.rate_steps, a.rate_warmup)
    if "robustness" in a.parts:
        out["robustness"] = bench_robustness(a.steps)
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
