"""Worker-side compute: batches in, gradients left in the flat gradient arenas.

Reference counterparts: ``DistributedWorker`` / ``CodedWorker`` / ``CyclicWorker`` (src/worker/baseline_worker.py:67-158,
rep_worker.py:63-155, cyclic_worker.py:63-163).  What is kept: one forward/backward per assigned sub-batch (1, or 2s+1
under the cyclic code), Prec@1/Prec@5/loss per step, local BatchNorm statistics, identical batches (and dropout /
augmentation randomness) for every holder of a batch.  What moved out: everything about communication -- encode,
adversary, compression and sends are the transport's business (parallel/fused_engine.py, collective_engine.py), not the
model's or the worker's.

One ``WorkerCompute`` serves *all* logical workers hosted by a process: they receive the same parameters, so they
share the model, its parameter arena and the gradient arenas, and differ only in the batches they are fed.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from ..config import JobConfig
from ..data import BatchPlan, TensorDataset, augment_cifar
from ..models import build_model
from ..ops import conv as _conv
from ..ops import dropout as _dropout
from ..ops import norm as _norm
from ..ops.loss import accuracy, cross_entropy_with_metrics  # noqa: F401  (accuracy re-exported)
from ..utils.metrics import wait_event
from .arena import ArenaLayout, ModelBinder


def plan_buckets(layout: ArenaLayout, nbuckets: int = 5):
    """Split the arena into contiguous tile ranges (whole tensors), returned in the order backprop finishes them (last
    layers first): ``[(tile_begin, tile_end, [param indices]), ...]``.  Cut points are at growing fractions of the bytes
    (35 / 65 / 85 / 95 % for 5 buckets): the early buckets are large (their transfer hides behind the rest of backprop),
    the final bucket -- the only one whose push is exposed after backprop ends -- is ~5 % of the model."""
    from .arena import TILE
    total = layout.ntiles
    fracs = {1: [], 2: [0.75], 3: [0.5, 0.9], 4: [0.4, 0.75, 0.95]}.get(nbuckets, [0.35, 0.65, 0.85, 0.95])
    cuts = [int(f * total) for f in fracs]
    buckets, cur, done_tiles = [], [], 0
    end_tile = total
    for i in range(layout.ntensors - 1, -1, -1):
        s = layout.specs[i]
        cur.append(i)
        done_tiles += (s.numel + TILE - 1) // TILE
        if cuts and done_tiles >= cuts[0] and i > 0:
            begin = s.offset // TILE
            buckets.append((begin, end_tile, cur))
            end_tile, cur = begin, []
            while cuts and done_tiles >= cuts[0]:
                cuts.pop(0)
    if cur:
        buckets.append((0, end_tile, cur))
    return buckets


def make_model(cfg: JobConfig) -> torch.nn.Module:
    torch.manual_seed(cfg.seed)
    kwargs = {}
    if cfg.num_classes != 10 and (cfg.network.startswith("ResNet") or cfg.network.startswith("VGG")):
        kwargs["num_classes"] = cfg.num_classes
    if cfg.dataset == "ImageNet" and cfg.network.startswith("ResNet"):
        # ImageNet-shaped ResNets (7x7 / stride-2 stem + max-pool, 224 x 224 inputs, 1000 classes)
        kwargs.update(num_classes=1000, imagenet_stem=True)
    return build_model(cfg.network, **kwargs)


class WorkerCompute:
    def __init__(self, cfg: JobConfig, device: torch.device, local_workers: List[int], plan: BatchPlan,
                 dataset: Optional[TensorDataset], layout: Optional[ArenaLayout] = None,
                 params_f32: Optional[torch.Tensor] = None, model: Optional[torch.nn.Module] = None):
        self.cfg, self.device, self.local_workers, self.plan, self.dataset = cfg, torch.device(device), local_workers, plan, dataset
        self.bf16 = cfg.dtype == "bf16" and self.device.type == "cuda"
        self.model = model if model is not None else make_model(cfg)
        self.channels_last = self.device.type == "cuda"
        self.layout = layout or ArenaLayout.from_model(self.model, self.bf16, self.channels_last)
        self.binder = ModelBinder(self.model, self.layout, self.device, self.bf16, params_f32)
        self.R = cfg.redundancy if cfg.approach == "cyclic" else 1
        # Zero-copy gradients (fused transport): autograd leaves every parameter's gradient wherever it allocated it and
        # the push kernel reads them through a device table of pointers -- no zero-fill, no accumulate-into-arena pass,
        # no gather (62 small kernels + 2 memsets per ResNet-18 backward otherwise).  The collective transports keep the
        # arena mode (p.grad = view of a zeroed flat arena).
        self.zero_copy = self.device.type == "cuda" and cfg.transport in ("nvl", "nccl_flat") and cfg.zero_copy_grads
        self.grads: List[Tuple[torch.Tensor, Optional[torch.Tensor]]] = \
            [] if self.zero_copy else [self.binder.new_grad_arenas() for _ in range(self.R)]
        T = self.layout.ntensors
        self.ptr_dev: Dict[int, torch.Tensor] = {}
        self.grad_refs: Dict[int, List[Optional[List[torch.Tensor]]]] = {}
        self._pinned_keep: List[torch.Tensor] = []
        if self.zero_copy:
            for wk in local_workers:
                self.ptr_dev[wk] = torch.zeros(self.R, T, dtype=torch.int64, device=self.device)
                self.grad_refs[wk] = [None] * self.R
        # gradient buckets (contiguous tile ranges, listed in the order backprop completes them) + readiness hooks:
        # the transport can ship a bucket while the remaining layers are still back-propagating
        self.buckets = plan_buckets(self.layout, 5)
        self._param_bucket = {i: b for b, (_, _, idxs) in enumerate(self.buckets) for i in idxs}
        self._bucket_left: List[int] = []
        self._bucket_cb = None
        # Gradient readiness comes from the MODEL's layer-wise backward driver (models/split.py: backward_normal fires
        # on_ready(param_index, param) as each gradient becomes final, reverse layer order -- the reference's "send layer l while
        # back-propagating layer l-1", resnet_split.py:431-623).  Models without the drivers get equivalent hooks here.
        self._has_drivers = all(hasattr(self.model, d) for d in ("backward_normal", "backward_coded", "backward_single"))
        if self._has_drivers:
            assert [id(p) for p in self.model._split_params()] == [id(p) for p in self.binder.params]
        else:
            for i, p in enumerate(self.binder.params):
                p.register_post_accumulate_grad_hook(self._make_ready_hook(i))
        self.model.train()
        self.has_dropout = any(isinstance(m, torch.nn.Dropout) for m in self.model.modules())
        c, h, w = self.model.input_shape if hasattr(self.model, "input_shape") else (3, 32, 32)
        if dataset is not None:
            c, h, w = dataset.images.shape[1:]
        B = cfg.batch_size
        self.x_u8: Dict[int, List[torch.Tensor]] = {}
        self.y: Dict[int, List[torch.Tensor]] = {}
        self.metrics: Dict[int, torch.Tensor] = {}
        # all sub-batches of this process live in ONE device buffer (and one pinned host buffer): a step's inputs travel as
        # a single H2D copy for the images and one for the labels instead of 2 per (worker, sub-batch)
        nsub = max(len(local_workers) * self.R, 1)
        self._x_all = torch.zeros(nsub, B, c, h, w, dtype=torch.uint8, device=self.device)
        self._y_all = torch.zeros(nsub, B, dtype=torch.long, device=self.device)
        for j, wk in enumerate(local_workers):
            self.x_u8[wk] = [self._x_all[j * self.R + k] for k in range(self.R)]
            self.y[wk] = [self._y_all[j * self.R + k] for k in range(self.R)]
            self.metrics[wk] = torch.zeros(3, dtype=torch.float32, device=self.device)   # loss, prec1, prec5
        self._pinned = None
        self._pin_slot = 0
        self._pin_events = [None, None]
        self._dataset_dev = None
        if dataset is not None:
            self._mean = dataset.mean.to(self.device)
            self._std = dataset.std.to(self.device)
        else:
            self._mean = torch.zeros(1, c, 1, 1, device=self.device)
            self._std = torch.ones(1, c, 1, 1, device=self.device)
        self.h2d_bytes = 0

    # ------------------------------------------------------------------ input staging
    def _ensure_pinned(self):
        if self._pinned is None:
            n = len(self.local_workers) * self.R
            shape = self.x_u8[self.local_workers[0]][0].shape
            pin = self.device.type == "cuda"
            self._pinned = [(torch.zeros((n,) + tuple(shape), dtype=torch.uint8, pin_memory=pin),
                             torch.zeros((n, shape[0]), dtype=torch.long, pin_memory=pin)) for _ in range(2)]

    def _native_loader(self):
        """The C++ gather/augment thread pool (csrc/host/dataload.cpp) when the dataset is an in-memory uint8 array."""
        if getattr(self, "_loader", None) is None and not getattr(self, "_loader_failed", False):
            try:
                from ..data.loader import NativeLoader
                d = self.dataset
                if (os.environ.get("DRACO_NATIVE_LOADER", "1") != "0" and d.images.dtype == torch.uint8 and d.images.dim() == 4
                        and d.images.is_contiguous() and d.labels.dtype == torch.int64 and d.labels.is_contiguous()):
                    self._loader = NativeLoader(d.images, d.labels, threads=2)
                else:
                    self._loader_failed = True
            except (OSError, RuntimeError, AttributeError):
                self._loader_failed = True
        return getattr(self, "_loader", None)

    def stage_batches(self, step: int) -> int:
        """Host -> device copy of every sub-batch this process needs at ``step``.  Returns bytes copied."""
        assert self.dataset is not None
        if self.cfg.data_on_device and self.device.type == "cuda":
            return self._stage_from_device(step)
        self._ensure_pinned()
        slot = self._pin_slot
        self._pin_slot ^= 1
        if self._pin_events[slot] is not None:
            wait_event(self._pin_events[slot])
        px, py = self._pinned[slot]
        aug = self.cfg.augment and self.dataset.name == "Cifar10"
        loader = self._native_loader()
        i = 0
        for wk in self.local_workers:
            ids = self.plan.batch_ids(step, wk)
            for k, idx in enumerate(self.plan.indices(step, wk)):
                # identical pixels for every holder of this (step, batch): the augmentation seed depends on those only
                seed = (self.cfg.seed * 7919 + step * 131 + ids[k]) if aug else None
                if loader is not None:
                    loader.submit(idx, px[i], py[i], seed=seed)      # C++ worker threads write the pinned staging memory
                else:
                    tidx = torch.from_numpy(np.ascontiguousarray(idx)).long()
                    if aug:
                        px[i].copy_(augment_cifar(self.dataset.images[tidx], seed))
                    else:
                        torch.index_select(self.dataset.images, 0, tidx, out=px[i])
                    torch.index_select(self.dataset.labels, 0, tidx, out=py[i])
                i += 1
        if loader is not None:
            loader.wait()
        nbytes = px.numel() + py.numel() * 8
        if self.device.type == "cuda":
            # The PCIe transfer runs on a COPY STREAM into device staging buffers while the compute stream still executes the
            # step that was enqueued before this call; the compute stream then only does a device-to-device copy (a few us)
            # into the buffers the captured step reads.  In-stream H2D copies would leave the GPU idle for the transfer.
            main = torch.cuda.current_stream(self.device)
            if getattr(self, "_copy_stream", None) is None:
                self._copy_stream = torch.cuda.Stream(device=self.device)
                self._x_stage, self._y_stage = torch.empty_like(self._x_all), torch.empty_like(self._y_all)
                self._stage_free = torch.cuda.Event()        # staging buffers consumed by the last D2D
                self._stage_full = torch.cuda.Event()
                self._stage_free.record(main)
            cs = self._copy_stream
            cs.wait_event(self._stage_free)
            with torch.cuda.stream(cs):
                self._x_stage.copy_(px, non_blocking=True)
                self._y_stage.copy_(py, non_blocking=True)
                ev = self._pin_events[slot] or torch.cuda.Event(blocking=True)
                ev.record(cs)                                # pinned slot reusable (host waits on it two stagings later)
                self._pin_events[slot] = ev
                self._stage_full.record(cs)
            main.wait_event(self._stage_full)
            self._x_all.copy_(self._x_stage, non_blocking=True)
            self._y_all.copy_(self._y_stage, non_blocking=True)
            self._stage_free.record(main)
        else:
            self._x_all.copy_(px)
            self._y_all.copy_(py)
        self.h2d_bytes = nbytes
        return nbytes

    def _stage_from_device(self, step: int) -> int:
        if self._dataset_dev is None:
            self._dataset_dev = (self.dataset.images.to(self.device), self.dataset.labels.to(self.device))
        imgs, labels = self._dataset_dev
        nbytes = 0
        for wk in self.local_workers:
            for k, idx in enumerate(self.plan.indices(step, wk)):
                tidx = torch.from_numpy(np.ascontiguousarray(idx)).long().to(self.device, non_blocking=True)
                torch.index_select(imgs, 0, tidx, out=self.x_u8[wk][k])
                torch.index_select(labels, 0, tidx, out=self.y[wk][k])
                nbytes += tidx.numel() * 8
        self.h2d_bytes = nbytes
        return nbytes

    def load_batch(self, wk: int, k: int, x_u8: torch.Tensor, y: torch.Tensor) -> None:
        """Directly provide a batch (public-API path used by tests / custom loops)."""
        self.x_u8[wk][k].copy_(x_u8, non_blocking=True)
        self.y[wk][k].copy_(y, non_blocking=True)

    # ------------------------------------------------------------------ compute
    def _prep_input(self, x_u8: torch.Tensor) -> torch.Tensor:
        if (os.environ.get("DRACO_FUSED_PREP", "1") == "1" and x_u8.is_cuda and x_u8.dim() == 4 and x_u8.shape[1] <= 4
                and x_u8.is_contiguous() and self.channels_last):
            return self._prep_input_fused(x_u8)
        x = (x_u8.float().div_(255.0).sub_(self._mean)).div_(self._std)
        if self.bf16:
            x = x.to(torch.bfloat16)
        if self.channels_last and x.dim() == 4:
            x = x.contiguous(memory_format=torch.channels_last)
        return x

    def _prep_input_fused(self, x_u8: torch.Tensor) -> torch.Tensor:
        """uint8 NCHW -> normalised channels-last tensor in the compute dtype, one launch (csrc/cuda/prep_input.cu)."""
        import ctypes as C

        from .. import _native as N
        lib = N.cuda()
        if not getattr(lib, "_prep_ready", False):
            lib.drc_prep_input.argtypes = [N.ptr, N.ptr, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float)] + [C.c_int] * 4 + [N.ptr]
            lib.drc_prep_input.restype = C.c_int
            lib._prep_ready = True
        n, c, h, w = x_u8.shape
        if getattr(self, "_prep_consts", None) is None:       # host copies of mean / std, read once (never under capture)
            m = self._mean.flatten().float().cpu().tolist()
            sd = self._std.flatten().float().cpu().tolist()
            m, sd = (m * c)[:c] if len(m) == 1 else m, (sd * c)[:c] if len(sd) == 1 else sd
            self._prep_consts = ((C.c_float * 4)(*(m + [0.0] * (4 - c))), (C.c_float * 4)(*(sd + [1.0] * (4 - c))))
        dt = torch.bfloat16 if self.bf16 else torch.float32
        out = torch.empty((n, c, h, w), dtype=dt, device=x_u8.device, memory_format=torch.channels_last)
        N.check(lib.drc_prep_input(x_u8.data_ptr(), out.data_ptr(), int(self.bf16), self._prep_consts[0], self._prep_consts[1],
                                   n, c, h, w, torch.cuda.current_stream().cuda_stream), "prep_input")
        return out

    def _on_grad_ready(self, i: int, _param=None) -> None:
        """Parameter ``i``'s gradient is final: when it completes a bucket, hand the bucket to the transport."""
        cb = self._bucket_cb
        if cb is None:
            return
        b = self._param_bucket[i]
        self._bucket_left[b] -= 1
        if self._bucket_left[b] == 0:
            cb(b)

    def _make_ready_hook(self, i: int):
        return lambda _param: self._on_grad_ready(i)

    def _dropout_step(self, step_host: Optional[int]):
        """Step source of the dropout key: the engine's device step counter when there is one (``self.step_dev``, set by the
        engine; required under graph capture), else a private device tensor refreshed from the host step, or the int on CPU."""
        if self.device.type != "cuda":
            return int(step_host or 1)
        if getattr(self, "step_dev", None) is not None:
            return self.step_dev
        assert step_host is not None, "dropout under graph capture needs the engine's device step counter"
        if getattr(self, "_step_priv", None) is None:
            self._step_priv = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._step_priv.fill_(int(step_host))
        return self._step_priv

    def forward_backward(self, wk: int, step_host: Optional[int] = None, on_bucket=None) -> None:
        """Run fwd/bwd for all sub-batches of logical worker ``wk``; gradients land in ``self.grads[k]``.
        Everything enqueued here is capturable in a CUDA graph (no host sync).  ``on_bucket(b)`` is called (from the
        autograd thread, on the backward stream) as soon as every gradient of bucket ``b`` is final -- only during the
        last sub-batch, i.e. when the values in the arenas are what will be sent."""
        met = self.metrics[wk]
        met.zero_()
        ids = self.plan.batch_ids(step_host or 1, wk) if self.has_dropout else None
        if self.zero_copy and not torch.cuda.is_current_stream_capturing():
            self._pinned_keep.clear()
        for k in range(self.R):
            if self.zero_copy:
                for p in self.binder.params:
                    p.grad = None
            else:
                g32, g16 = self.grads[k]
                g32.zero_()
                if g16 is not None:
                    g16.zero_()
                self.binder.bind_grads(g32, g16)
            if self.has_dropout:
                # identical dropout masks for every holder of this (step, batch): the mask is a hash of (seed, step, batch id, ...)
                # and on CUDA the step is read from device memory by the kernel, so a replayed graph advances by itself
                _dropout.set_context(self._dropout_step(step_host), self.cfg.seed, ids[k])
            x = self._prep_input(self.x_u8[wk][k])
            y = self.y[wk][k]
            with _norm.deferred_batch_counts():             # one multi-tensor kernel for all num_batches_tracked bumps
                out = self.model(x)
            loss = cross_entropy_with_metrics(out, y, met, 1.0 / self.R)      # also accumulates loss / Prec@1 / Prec@5
            if on_bucket is not None and k == self.R - 1:
                self._bucket_left = [len(idxs) for _, _, idxs in self.buckets]
                self._bucket_cb = on_bucket
            try:
                if not self._has_drivers:
                    loss.backward()                                      # permanent hooks (registered in __init__) report readiness
                elif self._bucket_cb is not None:
                    self.model.backward_normal(loss, on_ready=self._on_grad_ready)     # send-as-you-go: buckets leave during backward
                elif self.R > 1 and k < self.R - 1:
                    self.model.backward_coded(loss)                      # coded workers: collect, the encode happens after the last one
                else:
                    self.model.backward_single(loss)
            finally:
                self._bucket_cb = None
                if self.has_dropout:
                    _dropout.clear_context()
            if self.device.type == "cuda":
                _conv.join_wgrad_stream(self.device)         # weight gradients computed on the side stream (ops/conv.py) are final
            if self.zero_copy:
                self.grad_ptrs(0, self.layout.ntensors)          # validate dtype / strides against the arena layout
                self.grad_refs[wk][k] = [p.grad for p in self.binder.params]

    # ------------------------------------------------------------------ zero-copy pointer tables
    def grad_ptrs(self, lo: int, hi: int) -> List[int]:
        """Device addresses of the (current) gradients of parameters ``lo..hi-1``, validated against the arena layout."""
        out = []
        for i in range(lo, hi):
            p = self.binder.params[i]
            g = p.grad
            spec = self.layout.specs[i]
            assert g is not None, f"no gradient for {spec.name}"
            want = torch.bfloat16 if (self.bf16 and spec.is_bf16) else torch.float32
            if g.dtype != want or g.stride() != p.stride():
                # keep the arena element order: same dtype and the same (dense) strides as the parameter view
                g2 = torch.empty_strided(p.shape, p.stride(), dtype=want, device=g.device)
                g2.copy_(g)
                p.grad = g = g2
            out.append(g.data_ptr())
        return out

    def upload_ptrs(self, wk: int, k: int, lo: int, hi: int) -> None:
        """Enqueue (current stream) the H2D copy of table entries ``[lo, hi)`` of sub-batch ``k`` of worker ``wk``.
        Under graph capture only the validation runs: the table is filled once after the capture (addresses of
        captured allocations are stable across replays)."""
        ptrs = self.grad_ptrs(lo, hi)
        if torch.cuda.is_current_stream_capturing():
            return
        host = torch.tensor(ptrs, dtype=torch.int64).pin_memory()
        self._pinned_keep.append(host)
        self.ptr_dev[wk][k, lo:hi].copy_(host, non_blocking=True)

    def upload_all_ptrs(self, wk: int) -> None:
        """Table of worker ``wk`` from the references kept by the last forward_backward (after a graph capture)."""
        rows = []
        for k in range(self.R):
            refs = self.grad_refs[wk][k]
            rows.append([g.data_ptr() for g in refs])
        self.ptr_dev[wk].copy_(torch.tensor(rows, dtype=torch.int64))

    def flat_gradient(self, k: int = 0, wk: Optional[int] = None) -> torch.Tensor:
        """fp32 flat gradient of sub-batch k (collective transports; the fused push reads gradients in place)."""
        if self.zero_copy:
            refs = self.grad_refs[wk if wk is not None else self.local_workers[0]][k]
            out = self.layout.new_arena(self.device)
            for i, g in enumerate(refs):
                self.layout.view(out, i).copy_(g)
            return out
        g32, g16 = self.grads[k]
        return self.binder.flat_grad_f32(g32, g16)

    # ------------------------------------------------------------------ evaluation
    @torch.no_grad()
    def evaluate(self, dataset: TensorDataset, batch_size: int = 100, max_batches: Optional[int] = None) -> Dict[str, float]:
        """Test loss / Prec@1 / Prec@5 (reference: baseline_worker.py:275-293)."""
        was_training = self.model.training
        self.model.eval()
        tot, n = torch.zeros(3, device=self.device), 0
        mean, std = dataset.mean.to(self.device), dataset.std.to(self.device)
        for b, s in enumerate(range(0, len(dataset), batch_size)):
            if max_batches is not None and b >= max_batches:
                break
            xb = dataset.images[s:s + batch_size].to(self.device)
            yb = dataset.labels[s:s + batch_size].to(self.device)
            x = (xb.float() / 255.0 - mean) / std
            if self.bf16:
                x = x.to(torch.bfloat16)
            if self.channels_last:
                x = x.contiguous(memory_format=torch.channels_last)
            out = self.model(x)
            p1, p5 = accuracy(out, yb)
            tot += torch.stack([F.cross_entropy(out.float(), yb), p1, p5]) * xb.shape[0]
            n += xb.shape[0]
        self.model.train(was_training)
        tot = (tot / max(n, 1)).tolist()
        return {"loss": tot[0], "prec1": tot[1], "prec5": tot[2]}
