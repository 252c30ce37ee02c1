"""Public training API.

    cfg = JobConfig(network="ResNet18", dataset="Cifar10", approach="maj_vote", mode="maj_vote", group_size=3, ...)
    trainer = Trainer(cfg)                 # under torchrun: one process per GPU; standalone: single process
    for _ in range(cfg.max_steps):
        metrics = trainer.train_step()     # stages the batch (pinned H2D), runs the step, reads the loss back
    trainer.close()

``Trainer.fit()`` is the reference's ``master.start()`` + ``worker.train()`` pair (src/distributed_nn.py:87-133) in one
call: step loop, logging with the reference's fields, periodic evaluation + checkpoint every ``eval_freq`` steps,
resume from ``--checkpoint-step``.
"""
from __future__ import annotations

import os
import time
from typing import Dict, Optional

import torch
import torch.distributed as dist

from ..config import JobConfig
from ..data import TensorDataset, class_histograms, load_dataset
from ..utils.checkpoint import (arena_tensors, check_cc_center, check_mimic_state, check_worker_momentum, checkpoint_path,
                                load_checkpoint, model_buffers, restore_into, restore_worker_momentum, save_checkpoint)
from ..utils.metrics import MetricsLogger


def init_distributed(transport: str) -> tuple:
    """(rank, world, local_rank) from the torchrun environment; initialises the bootstrap process group."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        oversubscribed = torch.cuda.is_available() and world > torch.cuda.device_count()
        if transport == "gloo" or not torch.cuda.is_available() or oversubscribed or os.environ.get("DRACO_BOOTSTRAP") == "gloo":
            # Gloo-only bootstrap: CPU jobs, and GPU jobs with more processes than GPUs (several ranks share a device: NCCL
            # refuses duplicate devices, while the fused transport only needs object exchange + barriers from the process group
            # -- peer memory between two processes on ONE GPU works through the same VMM fd export/import)
            dist.init_process_group("gloo", rank=rank, world_size=world)
        else:
            torch.cuda.set_device(local)
            dist.init_process_group("cpu:gloo,cuda:nccl", rank=rank, world_size=world,
                                    device_id=torch.device("cuda", local))
    return rank, world, local


class Trainer:
    def __init__(self, cfg: JobConfig, rank: Optional[int] = None, world: Optional[int] = None,
                 device: Optional[torch.device] = None, dataset: Optional[TensorDataset] = None,
                 test_set: Optional[TensorDataset] = None, quiet: bool = False):
        if rank is None or world is None:
            rank, world, local = init_distributed(cfg.transport)
        else:
            local = rank
        self.rank, self.world = rank, world
        cfg.resolve(world)
        self.cfg = cfg
        if device is None:
            device = torch.device("cpu") if cfg.transport == "gloo" or not torch.cuda.is_available() \
                else torch.device("cuda", local % max(torch.cuda.device_count(), 1))
        self.device = torch.device(device)
        if self.device.type == "cuda":
            torch.cuda.set_device(self.device)
        if dataset is None:
            dataset = load_dataset(cfg.dataset, cfg.data_root, True, cfg.synthetic_size)
            if self.device.type == "cuda" and not cfg.data_on_device:
                dataset.pin()
        self.dataset, self.test_set = dataset, test_set
        # process-wide kernel switches owned by the fused engine: a later Trainer of another transport in the same process must not
        # inherit them (weight gradients on a side stream need the fused engine's stolen gradients and joins)
        from ..ops import conv as _conv_ops
        _conv_ops.WGRAD_SIDE_STREAM = False
        if cfg.transport == "nvl" and self.device.type == "cuda":
            from .fused_engine import FusedEngine
            self.engine = FusedEngine(cfg, rank, world, self.device, dataset)
        elif cfg.transport == "nccl_flat" and self.device.type == "cuda":
            from .flat_engine import FlatNcclEngine
            self.engine = FlatNcclEngine(cfg, rank, world, self.device, dataset)
        else:
            from .collective_engine import CollectiveEngine
            self.engine = CollectiveEngine(cfg, rank, world, self.device, dataset)
        self.logger = MetricsLogger(cfg.metrics_file, rank, cfg.log_interval, quiet)
        plan = getattr(getattr(self.engine, "worker", None), "plan", None)
        if plan is not None and plan.shards is not None:    # --dirichlet-alpha: every holder's class counts, once
            self.logger.log(0, "data", class_hist=class_histograms(dataset.labels.numpy(), plan.shards))
        self.is_ps = rank == 0
        self.eval_rank = self.engine.place.proc_of[1]          # the process hosting worker 1 evaluates (reference: rank 1)
        if cfg.checkpoint_step > 0:
            self.resume(cfg.checkpoint_step)

    # ------------------------------------------------------------------ stepping
    @property
    def step(self) -> int:
        return self.engine.step

    def train_step(self) -> Dict[str, float]:
        """One synchronous step through the public API: pinned-host batch -> device, step, loss back to host."""
        self.engine.train_step(stage=True)
        return self.engine.read_metrics()

    def train_step_pipelined(self) -> Optional[Dict[str, float]]:
        """One step through the public API with a *pipelined* result read: this step's inputs go pinned-host -> device,
        the step is enqueued, the D2H copy of its loss / Prec@k is enqueued behind it, and the metrics of the PREVIOUS
        step are returned (``None`` on the first call).  Every step's result is still read by the host -- one step late --
        but the GPU never idles waiting for the host to look at a loss.  ``drain()`` returns the last one."""
        eng = self.engine
        if hasattr(eng, "prefetch_inputs"):
            eng.train_step(stage=True, prefetch=False)
            handle = eng.enqueue_metrics_read()            # the small D2H copies go first: they would queue behind the input H2D
            eng.prefetch_inputs()
        else:
            eng.train_step(stage=True)
            handle = eng.enqueue_metrics_read()
        prev, self._pending = getattr(self, "_pending", None), (self.engine.step - 1, handle)
        return self.engine.resolve_metrics(prev[1]) if prev is not None else None

    def drain(self) -> Optional[Dict[str, float]]:
        prev, self._pending = getattr(self, "_pending", None), None
        return self.engine.resolve_metrics(prev[1]) if prev is not None else None

    def train_step_async(self, stage: bool = True) -> None:
        self.engine.train_step(stage=stage)

    def synchronize(self) -> None:
        self.engine.synchronize()

    # ------------------------------------------------------------------ loop
    def fit(self, max_steps: Optional[int] = None) -> Dict[str, float]:
        cfg = self.cfg
        last: Dict[str, float] = {}
        end = (max_steps or cfg.max_steps)
        while self.engine.step <= end:
            step = self.engine.step
            t0 = time.perf_counter()
            prev = self.train_step_pipelined()              # metrics of step-1 (None right after a drain)
            dt = time.perf_counter() - t0
            if self._log_step(step - 1, prev, dt):
                last = prev
            if step % cfg.eval_freq == 0 or step == end:
                cur = self.drain()                          # checkpoint / end of run: wait for the step just enqueued
                if self._log_step(step, cur, dt):
                    last = cur
                if step % cfg.eval_freq == 0:
                    self.checkpoint_and_eval(step)
        return last

    def _log_step(self, step: int, m: Optional[Dict[str, float]], dt: float) -> bool:
        if m is None:
            return False
        if "loss" in m:
            self.logger.log(step, "worker", t_step=dt, **m)
        if self.is_ps:
            self.logger.log(step, "ps", t_step=dt, **{k: v for k, v in m.items() if k.startswith("t_")})
        return "loss" in m

    # ------------------------------------------------------------------ eval / checkpoint
    def evaluate(self, max_batches: Optional[int] = None) -> Dict[str, float]:
        if self.test_set is None:
            self.test_set = load_dataset(self.cfg.dataset, self.cfg.data_root, False, self.cfg.synthetic_size)
        return self.engine.worker.evaluate(self.test_set, self.cfg.test_batch_size, max_batches)

    def checkpoint_and_eval(self, step: int) -> None:
        eng = self.engine
        eng.synchronize()
        if self.rank == self.eval_rank:
            res = self.evaluate(max_batches=20)
            self.logger.log(step, "eval", **res)
            if not self.logger.quiet:
                print("Testset Performance: Cur Step:{} Prec@1: {:.3f} Prec@5: {:.3f} Loss: {:.4f}".format(
                    step, res["prec1"], res["prec5"], res["loss"]), flush=True)
        # parameters after `step` updates live on the PS; BN statistics on the evaluating worker
        bufs = model_buffers(eng.worker.model) if self.rank == self.eval_rank else None
        if self.world > 1 and self.eval_rank != 0:
            box = [bufs if self.rank == self.eval_rank else None]
            if self.rank in (0, self.eval_rank):
                pass
            dist.broadcast_object_list(box, src=self.eval_rank)
            bufs = box[0]
        wmom = self._gather_worker_momentum() if self.cfg.worker_momentum > 0 else None
        if self.is_ps:
            ps = getattr(eng, "ps", None)
            mom = getattr(ps, "momentum", None)
            save_checkpoint(checkpoint_path(self.cfg.train_dir, step), eng.layout, eng.master_params(), mom, step,
                            self.cfg, bufs, opt_state=getattr(ps, "opt_state", None), worker_momentum=wmom)

    def _gather_worker_momentum(self) -> Dict[int, Dict[str, torch.Tensor]]:
        """Every logical worker's momentum, per tensor on the CPU (complete on the PS).  Each process converts its local
        workers'; in a multi-process job every worker process then broadcasts them, the way the BatchNorm statistics travel
        (every process takes part in each broadcast)."""
        eng = self.engine
        out = {w: arena_tensors(eng.layout, m) for w, m in eng.worker_momentum.items()}
        if self.world > 1:
            for p in range(1, self.world):
                if not eng.place.local_workers(p):
                    continue
                box = [out if self.rank == p else None]
                dist.broadcast_object_list(box, src=p)
                if self.rank == 0:
                    out.update(box[0])
        return out
    def resume(self, step: int) -> None:
        blob = load_checkpoint(checkpoint_path(self.cfg.train_dir, step))
        check_worker_momentum(blob, self.cfg.worker_momentum)
        check_cc_center(blob, self.cfg.mode == "centered_clip")
        check_mimic_state(blob, self.cfg.err_mode == "mimic")
        eng = self.engine
        if self.cfg.worker_momentum > 0:
            restore_worker_momentum(blob, eng.layout, eng.worker_momentum)       # every process: its own local workers
        ps = getattr(eng, "ps", None)
        if self.is_ps and hasattr(ps, "load_momentum"):
            # library-op PS: the momentum lives in the optimizer's state, rebuild it from the checkpoint
            dev = eng.master_params().device
            arena = eng.layout.new_arena(dev) if blob.get("momentum") else None
            extra = {k: eng.layout.new_arena(dev) for k, v in (blob.get("opt_state") or {}).items() if v}
            restore_into(blob, eng.layout, eng.master_params(), arena, extra)
            if hasattr(ps, "load_opt_state"):
                ps.load_opt_state(extra, step)              # before load_momentum: creates the Adam state entries
            if arena is not None:
                ps.load_momentum(arena)
        else:
            mom = getattr(ps, "momentum", None)
            restore_into(blob, eng.layout, eng.master_params(), mom if self.is_ps else None,
                         getattr(ps, "opt_state", None) if self.is_ps else None)
        if blob.get("buffers") and eng.worker is not None:
            eng.worker.model.load_state_dict(blob["buffers"], strict=False)
        eng.step = step + 1
        if hasattr(eng, "step_dev"):
            eng.step_dev.fill_(step + 1)
            eng._initial_broadcast()
        if hasattr(eng, "worker") and eng.worker is not None:
            eng.worker.binder.refresh_compute_copy()

    def close(self) -> None:
        self.engine.synchronize()
        self.engine.close()
        self.logger.close()
