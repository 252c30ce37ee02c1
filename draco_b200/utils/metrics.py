"""Metrics / logging / timing.

The reference prints ``time.time()`` deltas per step (worker: ``Time Cost / Comp / Comm / Encode / Prec@1 / Prec@5``,
src/worker/cyclic_worker.py:154-156; PS: ``Method Time Cost / Update Time Cost``, src/master/cyclic_master.py:143) and
nothing else.  Here: a human line with the same fields, JSONL records for machines, CUDA-event phase timers (device time,
reduced as max over ranks by the caller), and NVTX ranges around the phases so ``ncu``/profilers see the same names.
"""
from __future__ import annotations

import contextlib
import json
import subprocess
import threading
import time
from typing import Dict, List, Optional

import torch


def wait_event(event) -> None:
    """Host wait for a CUDA event created with ``blocking=True`` (cudaEventBlockingSync): the thread sleeps instead of
    spinning.  A host that burns CPU while the GPU works -- a spinning sync plus idle OpenMP workers spinning after every
    `index_select` of the input staging -- can run into a container's CPU quota and be descheduled for tens of milliseconds,
    which idles the GPU in any loop that reads results per step (`tools/diag_e2e.py` shows the effect)."""
    event.synchronize()


def limit_host_threads() -> None:
    """One process drives one GPU; its CPU work is the input gather (a few hundred KB per step).  Unless the user chose
    otherwise (OMP_NUM_THREADS), keep intra-op parallelism at one thread so that no pool of spinning OpenMP workers eats
    the CPU quota (torchrun does the same for multi-process launches)."""
    import os
    if "OMP_NUM_THREADS" not in os.environ:
        torch.set_num_threads(1)


class MetricsLogger:
    def __init__(self, path: Optional[str] = None, rank: int = 0, log_interval: int = 10, quiet: bool = False):
        self.rank, self.log_interval, self.quiet = rank, max(log_interval, 1), quiet
        self._fh = open(path.replace("{rank}", str(rank)), "a") if path else None

    def log(self, step: int, role: str, **fields) -> None:
        rec = {"ts": time.time(), "rank": self.rank, "role": role, "step": step, **fields}
        if self._fh:
            self._fh.write(json.dumps(rec) + "\n")
            self._fh.flush()
        if not self.quiet and step % self.log_interval == 0:
            f = fields.get
            if role == "worker":
                comp = f("t_comp", f("t_comp_encode_push", 0.0))
                print("Worker: {}, Step: {}, Loss: {:.4f}, Time Cost: {:.4f}, Comp: {:.4f}, Comm: {:.4f}, Encode: {:.4f}, "
                      "Prec@1: {:.2f}, Prec@5: {:.2f}".format(self.rank, step, f("loss", float("nan")), f("t_step", 0.0), comp,
                                                              f("t_fetch", 0.0) + f("t_comm", 0.0), f("t_encode", 0.0),
                                                              f("prec1", float("nan")), f("prec5", float("nan"))), flush=True)
            elif role == "ps":
                print("Master Step: {}, Method Time Cost: {:.6f}, Update Time Cost: {:.6f}".format(
                    step, f("t_decode", f("t_gather_decode_update_bcast", 0.0)), f("t_update", 0.0)), flush=True)

    def close(self) -> None:
        if self._fh:
            self._fh.close()
            self._fh = None


class PhaseTimer:
    """CUDA-event (or wall-clock on CPU) timers for named phases; ``elapsed()`` synchronises once."""

    def __init__(self, cuda: bool):
        self.cuda = cuda and torch.cuda.is_available()
        self._open: Dict[str, object] = {}
        self._pairs: List = []

    @contextlib.contextmanager
    def phase(self, name: str):
        if self.cuda:
            torch.cuda.nvtx.range_push(name)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            try:
                yield
            finally:
                e.record()
                torch.cuda.nvtx.range_pop()
                self._pairs.append((name, s, e))
        else:
            t0 = time.perf_counter()
            try:
                yield
            finally:
                self._pairs.append((name, t0, time.perf_counter()))

    def elapsed(self) -> Dict[str, float]:
        out: Dict[str, float] = {}
        if self.cuda:
            torch.cuda.synchronize()
        for name, s, e in self._pairs:
            dt = s.elapsed_time(e) / 1e3 if self.cuda else e - s
            out[name] = out.get(name, 0.0) + dt
        self._pairs.clear()
        return out


class ClockSampler:
    """Samples SM clocks / throttle reasons with nvidia-smi while a timed region runs (bench.py contract)."""

    QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int = 0, period_ms: int = 100):
        self.gpu_index, self.period_ms = gpu_index, period_ms
        self.proc: Optional[subprocess.Popen] = None
        self.lines: List[str] = []
        self._thread: Optional[threading.Thread] = None

    def start(self) -> None:
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.QUERY}", "--format=csv,noheader,nounits",
                                          "-i", str(self.gpu_index), "-lms", str(self.period_ms)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None
            return

        def pump():
            for line in self.proc.stdout:
                self.lines.append(line.strip())
        self._thread = threading.Thread(target=pump, daemon=True)
        self._thread.start()

    def stop(self) -> Dict[str, object]:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except subprocess.TimeoutExpired:
            self.proc.kill()
        sm, smax, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            parts = [p.strip() for p in ln.split(",")]
            if len(parts) < 8:
                continue
            try:
                sm.append(float(parts[1])); smax.append(float(parts[2]))
            except ValueError:
                continue
            for nm, v in zip(names, parts[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "reasons": sorted(reasons), "samples": len(sm)}
