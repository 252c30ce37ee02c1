"""Measure adaptive robust clipping (``--arc tensor | model``) on one GPU and print one JSON line.

(a) ``kernels``: device time of csrc/cuda/arc.cu on the ResNet-18 arena at P = 7, 15 and 16 (f = 1, 3, 3): the norm pass, the
    factors, the scale pass, the tensor-scope chain and the model-scope chain (CUDA events, median of 3 rounds).  The bytes the
    algorithm needs are P rows of slab read by the norm and 2k rows read and written by the scale, with k counted from the
    factors the data gave; their rate is set against the H100 SXM's 3.35 TB/s.
(b) ``step_rate``: device-timed steps/s of bench.py's job (ResNet-18 / CIFAR-10, batch 128, bf16, captured graph) at 15 workers
    and ``--worker-fail 3`` under rev_grad, for normal, coordinate_median, multi_krum, centered_clip and nnm/coordinate_median,
    each without ARC, with ``--arc tensor`` and with ``--arc model``, with the kernels launched per step and whether the PS
    pipelines.  Every arm runs in its own process; the arms alternate over --rate-rounds.
(c) ``loss``: final training loss after --steps steps, 15 workers, 3 liars: the plain mean with and without ``--arc tensor``
    under the default rev_grad liars, and coordinate_median / multi_krum with and without ``--arc tensor`` under alie, minmax
    and mimic, with IID data and with --dirichlet-alpha 0.1.  Single short runs on synthetic data.

    python tools/bench_arc.py [--parts kernels rate loss] [--out FILE]
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

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet
RATE_ARMS = tuple((approach, mode, arc) for approach, mode in (("baseline", "normal"), ("baseline", "coordinate_median"),
                                                               ("baseline", "multi_krum"), ("baseline", "centered_clip"),
                                                               ("nnm", "coordinate_median"))
                  for arc in (None, "tensor", "model"))
LOSS_ATTACKS = ("alie", "minmax", "mimic")


def gpu_info() -> dict:
    """Card name, power limit and max SM clock, read in the same call as the measurement."""
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_max_sm_clock_sm_clock"] = q.stdout.strip()
    except Exception as e:          # the measurement still stands; the card's limits are then unknown
        info["power_limit_max_sm_clock_sm_clock"] = f"unavailable: {e}"
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
    from draco_b200.codes.oracle import arc_k
    from draco_b200.models import build_model
    from draco_b200.ops import kernels as K
    from draco_b200.parallel.arena import ArenaLayout
    dev = torch.device("cuda", 0)
    L = ArenaLayout.from_model(build_model("ResNet18", num_classes=10), bf16=True, channels_last=True)
    valid = torch.from_numpy(L.valid_mask()).to(dev).float()
    numel = int(valid.sum().item())
    res = []
    for P, f in ((7, 1), (15, 3), (16, 3)):
        k = arc_k(P, f)
        g = torch.Generator(device=dev).manual_seed(P)
        # one scale per (row, tensor), so every tensor clips its k largest rows and the scale pass has real work
        base = torch.randn(P, L.total, device=dev, generator=g) * valid
        for sp in L.specs:
            base[:, sp.offset: sp.offset + sp.numel] *= torch.rand(P, 1, device=dev, generator=g) * 4 + 0.1
        slab = base.clone()
        tws, mws = K.ArcWorkspace(L, P, dev, model=False), K.ArcWorkspace(L, P, dev, model=True)
        row = {"P": P, "f": f, "k": k, "slab_MB": round(P * numel * 4 / 1e6, 1)}
        row["norm_us"] = _time(lambda: K.arc_norm(L, slab, L.total, P, tws), iters)
        row["factors_us"] = _time(lambda: K.arc_factors(L, P, k, tws), iters)
        row["model_factors_us"] = _time(lambda: K.arc_model_factors(L, P, k, mws), iters)
        # the scale pass rewrites the slab, so each timed call starts from the same data: the copy is timed alone and taken off
        copy_us = _time(lambda: slab.copy_(base), iters)
        row["copy_us"] = copy_us
        K.arc_factors(L, P, k, tws)
        row["scale_us"] = round(_time(lambda: (slab.copy_(base), K.arc_scale(L, slab, L.total, P, tws)), iters) - copy_us, 2)
        row["tensor_chain_us"] = round(_time(lambda: (slab.copy_(base), K.arc_clip(L, slab, L.total, P, k, tws)), iters) - copy_us, 2)
        row["model_chain_us"] = round(_time(lambda: (slab.copy_(base), K.arc_clip(L, slab, L.total, P, k, mws)), iters) - copy_us, 2)
        for name, ws in (("tensor", tws), ("model", mws)):
            slab.copy_(base)
            K.arc_clip(L, slab, L.total, P, k, ws)
            clipped = (ws.factors < 1)                               # [T, P]: the (tensor, row) pairs the scale pass rewrites
            sizes = torch.tensor([sp.numel for sp in L.specs], device=dev, dtype=torch.float64)
            scaled = float((clipped.double().sum(1) * sizes).sum().item())
            need = (P * numel + 2 * scaled) * 4
            row[f"{name}_rows_clipped_per_tensor"] = round(float(clipped.sum().item()) / L.ntensors, 2)
            row[f"{name}_bytes_MB"] = round(need / 1e6, 1)
            t_us = row[f"{name}_chain_us"]
            row[f"{name}_TBps"] = round(need / (t_us * 1e-6) / 1e12, 2) if t_us > 0 else None
            row[f"{name}_share_of_3.35TBps"] = round(need / HBM_BYTES_PER_S / (t_us * 1e-6), 3) if t_us > 0 else None
        res.append(row)
    return res


def run_one(spec: dict) -> dict:
    import torch
    from draco_b200 import JobConfig
    from draco_b200.parallel.trainer import Trainer
    steps = spec["warmup"] + spec["steps"]
    cc = spec["mode"] == "centered_clip"
    cfg = JobConfig(network="ResNet18", dataset="Cifar10", approach=spec["approach"], mode=spec["mode"], batch_size=128,
                    num_workers=15, group_size=3, worker_fail=3, err_mode=spec["err_mode"], arc=spec["arc"],
                    dirichlet_alpha=spec.get("alpha"), lr=0.01, momentum=0.9, clip_tau=0.05 if cc else None,
                    max_steps=steps + 8, eval_freq=10 ** 9, transport="nvl", dtype="bf16", cuda_graphs=True,
                    compress_grad="None", synthetic_size=8192, log_interval=10 ** 9)
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


def bench_rate(rounds: int, steps: int, warmup: int, rules) -> list:
    arms = tuple(arm for arm in RATE_ARMS if not rules or f"{arm[0]}/{arm[1]}" in rules)
    runs = {arm: [] for arm in arms}
    info, errors = {}, []
    for r in range(rounds):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            approach, mode, arc = arm
            o = spawn(dict(kind="rate", approach=approach, mode=mode, arc=arc, err_mode="rev_grad", steps=steps, warmup=warmup))
            if "error" in o:
                errors.append(o)
                continue
            runs[arm].append(round(o["steps_per_s"], 2))
            info[arm] = (o["kernels_per_step"], o["pipelined_ps"])
    res = []
    for arm, v in runs.items():
        k, pipe = info.get(arm, (None, None))
        res.append({"approach": arm[0], "mode": arm[1], "arc": arm[2], "steps_per_s": v,
                    "median": statistics.median(v) if v else None, "kernels_per_step": k, "pipelined_ps": pipe})
    return res + errors


def bench_loss(steps: int, alphas) -> list:
    res = []
    if None in alphas:
        for arc in (None, "tensor"):
            res.append(spawn(dict(kind="loss", approach="baseline", mode="normal", arc=arc, err_mode="rev_grad", steps=steps,
                                  warmup=0)))
    for alpha in alphas:
        for err in LOSS_ATTACKS:
            for mode in ("coordinate_median", "multi_krum"):
                for arc in (None, "tensor"):
                    res.append(spawn(dict(kind="loss", approach="baseline", mode=mode, arc=arc, err_mode=err, alpha=alpha,
                                          steps=steps, warmup=0)))
    return res


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--one", type=str, default=None, help=argparse.SUPPRESS)
    ap.add_argument("--parts", nargs="+", default=["kernels", "rate", "loss"], choices=("kernels", "rate", "loss"))
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rate-rounds", type=int, default=2)
    ap.add_argument("--rate-steps", type=int, default=30)
    ap.add_argument("--rate-warmup", type=int, default=5)
    ap.add_argument("--rate-rules", nargs="+", default=None, help="approach/mode arms to time (default: every arm)")
    ap.add_argument("--loss-alphas", nargs="+", default=["iid", "0.1"], help="iid and / or Dirichlet alphas of the loss runs")
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
        out["kernels"] = bench_kernels(a.iters)
    if "rate" in a.parts:
        out["step_rate"] = bench_rate(a.rate_rounds, a.rate_steps, a.rate_warmup, a.rate_rules)
    if "loss" in a.parts:
        out["loss"] = bench_loss(a.steps, [None if x == "iid" else float(x) for x in a.loss_alphas])
    out["gpu_after"] = gpu_info()
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
