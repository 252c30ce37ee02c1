"""Checkpoint / resume.

Reference behaviour: the PS pickles the whole module to ``train_dir + "model_step_" + step`` every
``eval_freq`` steps (src/master/baseline_master.py:237-243), worker 1 saves a state_dict for ResNets
(src/worker/baseline_worker.py:298-302), and resume exists only for the baseline approach from a hard-coded path without
optimizer state (baseline_master.py:54-57).

Here one file per checkpoint, same naming (``<train_dir>model_step_<N>``), containing logical (NCHW) parameter tensors,
the momentum buffers, the step, the BatchNorm statistics of the evaluating worker (the PS never runs a forward pass, so
its own BN statistics would be meaningless -- the reason the reference refuses to save ResNets on the PS) and the job
config.  Resume works for every approach and restores optimizer state.  With ``--worker-momentum`` the blob also holds
every logical worker's momentum (``"worker_momentum": {w: {tensor name: fp32 tensor}}``); the key is absent otherwise.  Under
``--mode centered_clip`` the PS's centre travels with the optimizer arenas as ``opt_state["cc_center"]``, and under
``--err-mode mimic`` the attack's running mean and direction as ``opt_state["mimic_m"]`` and ``["mimic_z"]``; other jobs have
no such entries.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch

from ..config import JobConfig
from ..parallel.arena import ArenaLayout


def checkpoint_path(train_dir: str, step: int) -> str:
    return f"{train_dir}model_step_{step}"


def save_checkpoint(path: str, layout: ArenaLayout, params: torch.Tensor, momentum: Optional[torch.Tensor], step: int,
                    cfg: JobConfig, buffers: Optional[Dict[str, torch.Tensor]] = None,
                    opt_state: Optional[Dict[str, torch.Tensor]] = None,
                    worker_momentum: Optional[Dict[int, Dict[str, torch.Tensor]]] = None) -> None:
    """``momentum``: SGD momentum buffer / Adam first moment arena; ``opt_state``: further optimizer arenas by name
    (Adam: ``exp_avg_sq``, AMSGrad: ``max_exp_avg_sq``) -- all saved per parameter tensor.  ``worker_momentum``: every
    logical worker's state as ``arena_tensors`` gives it (None: no worker momentum, no key)."""
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    state = {layout.specs[i].name: layout.view(params, i).detach().float().cpu().contiguous().clone()
             for i in range(layout.ntensors)}
    mom = None
    if momentum is not None:
        mom = {layout.specs[i].name: layout.view(momentum, i).detach().float().cpu().contiguous().clone()
               for i in range(layout.ntensors)}
    extra = {name: {layout.specs[i].name: layout.view(arena, i).detach().float().cpu().contiguous().clone()
                    for i in range(layout.ntensors)} for name, arena in (opt_state or {}).items() if arena is not None}
    blob = {"format": "draco_b200/1", "step": int(step), "state_dict": state, "momentum": mom, "opt_state": extra,
            "buffers": {k: v.detach().cpu().clone() for k, v in (buffers or {}).items()}, "config": cfg.to_dict()}
    if worker_momentum is not None:
        blob["worker_momentum"] = {int(w): dict(t) for w, t in sorted(worker_momentum.items())}
    tmp = path + ".tmp"
    torch.save(blob, tmp)
    os.replace(tmp, path)


def arena_tensors(layout: ArenaLayout, arena: torch.Tensor) -> Dict[str, torch.Tensor]:
    """{tensor name: fp32 CPU tensor in the logical (NCHW) shape} of one arena."""
    return {layout.specs[i].name: layout.view(arena, i).detach().float().cpu().contiguous().clone()
            for i in range(layout.ntensors)}


def check_worker_momentum(blob: dict, beta: float) -> None:
    """A job resumes only from a checkpoint of the same kind: with worker momentum iff the job runs with it."""
    has = "worker_momentum" in blob
    if beta > 0 and not has:
        raise ValueError(f"--worker-momentum {beta}: the checkpoint holds no worker momentum (it was written by a job without "
                         f"--worker-momentum), so the workers' state cannot be restored")
    if beta == 0 and has:
        raise ValueError("the checkpoint holds worker momentum (it was written with --worker-momentum): resume it with the same "
                         "--worker-momentum, or the workers' state would be dropped")


def check_cc_center(blob: dict, centered_clip: bool) -> None:
    """A job resumes only from a checkpoint of the same kind: with centered clipping's centre iff the job clips."""
    has = "cc_center" in (blob.get("opt_state") or {})
    if centered_clip and not has:
        raise ValueError("--mode centered_clip: the checkpoint holds no centre (it was written by a job with another rule), so "
                         "the clipping would restart around zero")
    if not centered_clip and has:
        raise ValueError("the checkpoint holds centered clipping's centre (it was written with --mode centered_clip): resume it "
                         "with the same --mode, or the centre would be dropped")


def check_mimic_state(blob: dict, mimic: bool) -> None:
    """A job resumes only from a checkpoint of the same kind: with the mimic attack's running mean and direction iff the job
    runs --err-mode mimic."""
    has = "mimic_m" in (blob.get("opt_state") or {}) and "mimic_z" in (blob.get("opt_state") or {})
    if mimic and not has:
        raise ValueError("--err-mode mimic: the checkpoint holds no mimic state (it was written by a job with another "
                         "--err-mode), so the attack's direction and running mean cannot be restored")
    if not mimic and "mimic_m" in (blob.get("opt_state") or {}):
        raise ValueError("the checkpoint holds the mimic attack's state (it was written with --err-mode mimic): resume it with "
                         "the same --err-mode, or the state would be dropped")


def restore_worker_momentum(blob: dict, layout: ArenaLayout, arenas: Dict[int, torch.Tensor]) -> None:
    """Copy the saved state of every worker in ``arenas`` (this process's local workers) into its arena."""
    saved = blob["worker_momentum"]
    with torch.no_grad():
        for w, arena in arenas.items():
            if w not in saved:
                raise ValueError(f"the checkpoint holds no worker momentum for worker {w} (it has workers {sorted(saved)})")
            for i, spec in enumerate(layout.specs):
                layout.view(arena, i).copy_(saved[w][spec.name])


def load_checkpoint(path: str) -> dict:
    blob = torch.load(path, map_location="cpu", weights_only=False)
    if blob.get("format") != "draco_b200/1":
        raise ValueError(f"{path}: not a draco_b200 checkpoint")
    return blob


def restore_into(blob: dict, layout: ArenaLayout, params: torch.Tensor, momentum: Optional[torch.Tensor],
                 opt_state: Optional[Dict[str, torch.Tensor]] = None) -> int:
    with torch.no_grad():
        for i, spec in enumerate(layout.specs):
            layout.view(params, i).copy_(blob["state_dict"][spec.name])
            if momentum is not None and blob.get("momentum"):
                layout.view(momentum, i).copy_(blob["momentum"][spec.name])
            for name, arena in (opt_state or {}).items():
                saved = (blob.get("opt_state") or {}).get(name)
                if arena is not None and saved:
                    layout.view(arena, i).copy_(saved[spec.name])
    return int(blob["step"])


def model_buffers(model: torch.nn.Module) -> Dict[str, torch.Tensor]:
    return {k: v for k, v in model.named_buffers()}


def load_into_model(blob: dict, model: torch.nn.Module) -> None:
    """Load a checkpoint into a plain (unbound) model, e.g. in the evaluator."""
    sd = dict(blob["state_dict"])
    sd.update(blob.get("buffers") or {})
    model.load_state_dict(sd, strict=False)
