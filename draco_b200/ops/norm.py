"""BatchNorm2d with fused residual-add + ReLU on the sm_90a kernels of ``csrc/cuda/bn_fused.cu``.

``FusedBatchNorm2d`` *is* an ``nn.BatchNorm2d`` (same parameters, buffers and state_dict keys as the reference's models,
src/model_ops/resnet.py:19-24) whose ``forward(x, residual=None, relu=False)`` computes
``relu?(batch_norm(x) + residual)``.  On CUDA, in training mode, for bf16 channels-last activations with a power-of-two
channel count it runs as streaming kernels with deterministic reductions (forward: apply only when the producing convolution's epilogue
delivered the statistics, else statistics + apply; backward: reduce + apply); everywhere else it is exactly ``F.batch_norm`` (+ add, + relu) so CPU runs and evaluation are unchanged.
``backend_counters`` records which path served each call.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from .. import _native as N

backend_counters = {"fused": 0, "aten": 0}
_counter_cache = {}


def _lib():
    lib = N.cuda()
    if not getattr(lib, "_bn_ready", False):
        st = N.ptr
        lib.drc_bn_supported.argtypes = [C.c_int]
        lib.drc_bn_supported.restype = C.c_int
        lib.drc_bn_workspace.argtypes = [N.i64, C.c_int, C.c_int]
        lib.drc_bn_workspace.restype = N.i64
        lib.drc_bn_fwd.argtypes = [N.ptr] * 12 + [N.i64, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, C.c_int, st]
        lib.drc_bn_fwd.restype = C.c_int
        lib.drc_bn_fwd_dual.argtypes = [N.ptr] * 12 + [N.i64, C.c_int, C.c_int, st]
        lib.drc_bn_fwd_dual.restype = C.c_int
        lib.drc_bn_bwd.argtypes = [N.ptr] * 15 + [N.i64, C.c_int, C.c_int, C.c_int, st]
        lib.drc_bn_bwd.restype = C.c_int
        lib.drc_bn_bwd_dual.argtypes = [N.ptr] * 20 + [N.i64, C.c_int, C.c_int, st]
        lib.drc_bn_bwd_dual.restype = C.c_int
        lib.drc_bn_bwd_apply.argtypes = [N.ptr] * 7 + [N.i64, C.c_int, C.c_int, st]
        lib.drc_bn_bwd_apply.restype = C.c_int
        lib._bn_ready = True
    return lib


# Set by the engine when logical workers run on concurrent streams: only one worker per process may update the shared
# running statistics.
UPDATE_RUNNING_STATS = True


# ``num_batches_tracked += 1`` is a kernel launch per BatchNorm layer per forward (20 launches per ResNet-18 step).  Inside ``deferred_batch_counts()`` the fused path only remembers the
# counters and the context exit bumps all of them with ONE multi-tensor kernel.
_defer_counts = False
_pending_counts: list = []


class deferred_batch_counts:
    def __enter__(self):
        global _defer_counts
        self._prev = _defer_counts
        _defer_counts = True
        return self

    def __exit__(self, *exc):
        global _defer_counts
        _defer_counts = self._prev
        if not _defer_counts and _pending_counts:
            pend = list(_pending_counts)
            _pending_counts.clear()
            torch._foreach_add_(pend, 1)
        return False


def _counter(device: torch.device) -> torch.Tensor:
    """Grid-barrier / last-CTA counters; one set per (device, stream) so that concurrent streams never share them."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    if key not in _counter_cache:
        _counter_cache[key] = torch.zeros(32, dtype=torch.int32, device=device)   # zero-filled on this very stream
    return _counter_cache[key]


def _sms(device: torch.device) -> int:
    return torch.cuda.get_device_properties(device).multi_processor_count


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


# ReLU mask modes of the backward kernels (csrc/cuda/bn_fused.cu, drc_bn_bwd)
MASK_NONE, MASK_Y, MASK_X, MASK_BITS = 0, 1, 2, 3


def _mask_mode(has_residual: bool) -> int:
    """``DRACO_BN_MASK``: ``bits`` (default) -- the forward stores one bit per element (M * C / 8 bytes) and the backward reads
    it instead of the saved output;  ``y`` -- the backward reads the saved output y;  ``x`` -- recomputed from x with the
    forward's own arithmetic (layers without a residual input; one saved activation less).  All three give the same mask."""
    mode = os.environ.get("DRACO_BN_MASK", "bits")
    if mode == "y":
        return MASK_Y
    if mode == "x" and not has_residual:
        return MASK_X
    return MASK_BITS


def _new_mask(x: torch.Tensor) -> torch.Tensor:
    n, c, h, w = x.shape
    return torch.empty(n * h * w * c // 8, dtype=torch.uint8, device=x.device)


def fused_supported(x: torch.Tensor, training: bool) -> bool:
    return (training and x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and
            x.is_contiguous(memory_format=torch.channels_last) and os.environ.get("DRACO_BN", "fused") == "fused" and
            bool(_lib().drc_bn_supported(x.shape[1])))


class _BnActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, gamma, beta, running_mean, running_var, eps, momentum, relu, mean, invstd, link_box=None):
        """``mean`` / ``invstd`` given: statistics came out of the producing convolution's epilogue, only the apply kernel runs."""
        lib = _lib()
        n, c, h, w = x.shape
        M = n * h * w
        dev = x.device
        y = torch.empty_like(x, memory_format=torch.channels_last)
        have_stats = mean is not None
        if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
            residual = residual.contiguous(memory_format=torch.channels_last)
        mode = _mask_mode(residual is not None) if relu else MASK_NONE
        mask = _new_mask(x) if mode == MASK_BITS else None
        if have_stats:
            ws_ptr = None
        else:
            mean = torch.empty(c, dtype=torch.float32, device=dev)
            invstd = torch.empty(c, dtype=torch.float32, device=dev)
            ws = torch.empty(int(lib.drc_bn_workspace(M, c, _sms(dev))), dtype=torch.float32, device=dev)
            ws_ptr = ws.data_ptr()
        N.check(lib.drc_bn_fwd(x.data_ptr(), _p(residual), y.data_ptr(), _p(mask), gamma.data_ptr(), beta.data_ptr(), _p(running_mean),
                               _p(running_var), mean.data_ptr(), invstd.data_ptr(), ws_ptr, _counter(dev).data_ptr(),
                               M, c, float(eps), float(momentum), int(relu), _sms(dev), int(have_stats),
                               torch.cuda.current_stream().cuda_stream), "bn_fwd")
        # ReLU mask in backward (see _mask_mode): the forward's bits by default -- y stays alive anyway as the next convolution's
        # saved input, so reading 1/16 of it as bits costs 1/16 of the bytes
        ctx.save_for_backward(x, y if mode == MASK_Y else mask, gamma, beta, mean, invstd)
        ctx.mode, ctx.has_res = mode, residual is not None
        ctx.link = None
        if link_box is not None:                       # see ops.conv.BnBwdLink: the consumer convolution may reduce for us
            from .conv import BnBwdLink
            ctx.link = link_box[0] = BnBwdLink(x, mean, invstd, relu)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = _lib()
        x, y_or_mask, gamma, beta, mean, invstd = ctx.saved_tensors
        n, c, h, w = x.shape
        M = n * h * w
        dev = x.device
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x, memory_format=torch.channels_last)
        link, ctx.link = ctx.link, None
        if link is not None and link.sums is not None and link.dz is not None and link.dz.data_ptr() == dy.data_ptr():
            # the consuming convolution's dgrad epilogue already masked dy (dz) and reduced sum(dz), sum(dz * xhat): apply only
            backend_counters["bwd_in_conv"] = backend_counters.get("bwd_in_conv", 0) + 1
            torch.cuda.set_device(dev)
            N.check(lib.drc_bn_bwd_apply(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
                                         link.sums.data_ptr(), dx.data_ptr(), M, c, _sms(dev),
                                         torch.cuda.current_stream().cuda_stream), "bn_bwd_apply")
            dgamma, dbeta = link.dgamma, link.dbeta
            link.dz = link.sums = None
            return dx, (dy if ctx.has_res else None), dgamma, dbeta, None, None, None, None, None, None, None, None
        dres = torch.empty_like(x, memory_format=torch.channels_last) if ctx.has_res else None
        dgamma = torch.empty(c, dtype=torch.float32, device=dev)
        dbeta = torch.empty(c, dtype=torch.float32, device=dev)
        torch.cuda.set_device(dev)
        sums = torch.empty(2 * c, dtype=torch.float32, device=dev)
        ws = torch.empty(int(lib.drc_bn_workspace(M, c, _sms(dev))), dtype=torch.float32, device=dev)
        y = y_or_mask if ctx.mode == MASK_Y else None
        mask = y_or_mask if ctx.mode == MASK_BITS else None
        N.check(lib.drc_bn_bwd(dy.data_ptr(), _p(y), _p(mask), x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), mean.data_ptr(),
                               invstd.data_ptr(), dx.data_ptr(), _p(dres), dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(),
                               sums.data_ptr(), _counter(dev)[8:].data_ptr(), M, c, ctx.mode, _sms(dev),
                               torch.cuda.current_stream().cuda_stream), "bn_bwd")
        return dx, dres, dgamma, dbeta, None, None, None, None, None, None, None, None


class _BnPairFn(torch.autograd.Function):
    """``relu(bn(x) + bn_s(xs))`` of a downsampling block in one pass each way: the forward never writes the shortcut layer's
    output, the backward never writes the masked gradient both layers share (it reduces both layers' sums in one pass over
    dy, x, xs and the ReLU bits, then writes dx and dxs).  Both layers' statistics came from their convolutions' epilogues.
    Every output, gradient and statistic equals the two-layer path's (``bn(x, residual=bn_s(xs), relu=True)``) bit for bit."""

    @staticmethod
    def forward(ctx, x, xs, gamma, beta, gamma_s, beta_s, mean, invstd, mean_s, invstd_s, link_box=None):
        lib = _lib()
        n, c, h, w = x.shape
        dev = x.device
        y = torch.empty_like(x, memory_format=torch.channels_last)
        mask = _new_mask(x)
        N.check(lib.drc_bn_fwd_dual(x.data_ptr(), xs.data_ptr(), y.data_ptr(), mask.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                    mean.data_ptr(), invstd.data_ptr(), gamma_s.data_ptr(), beta_s.data_ptr(), mean_s.data_ptr(),
                                    invstd_s.data_ptr(), n * h * w, c, _sms(dev), torch.cuda.current_stream().cuda_stream),
                "bn_fwd_dual")
        ctx.save_for_backward(x, xs, mask, gamma, beta, gamma_s, mean, invstd, mean_s, invstd_s)
        ctx.link = None
        if link_box is not None:
            from .conv import BnBwdLink
            ctx.link = link_box[0] = BnBwdLink(x, mean, invstd, True)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = _lib()
        x, xs, mask, gamma, beta, gamma_s, mean, invstd, mean_s, invstd_s = ctx.saved_tensors
        n, c, h, w = x.shape
        M = n * h * w
        dev = x.device
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        torch.cuda.set_device(dev)
        stream = torch.cuda.current_stream().cuda_stream
        dx = torch.empty_like(x, memory_format=torch.channels_last)
        dxs = torch.empty_like(xs, memory_format=torch.channels_last)
        dgamma, dbeta, dgamma_s, dbeta_s = (torch.empty(c, dtype=torch.float32, device=dev) for _ in range(4))
        sums = torch.empty(4 * c, dtype=torch.float32, device=dev)
        ws_floats = int(lib.drc_bn_workspace(M, c, _sms(dev)))
        link, ctx.link = ctx.link, None
        if link is not None and link.sums is not None and link.dz is not None and link.dz.data_ptr() == dy.data_ptr():
            # the consuming convolution's dgrad epilogue already masked dy (dz) and reduced the main layer's sums: apply it, then
            # the shortcut layer's reduce + apply over dz, as the two-layer path does
            backend_counters["bwd_in_conv"] = backend_counters.get("bwd_in_conv", 0) + 1
            N.check(lib.drc_bn_bwd_apply(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
                                         link.sums.data_ptr(), dx.data_ptr(), M, c, _sms(dev), stream), "bn_bwd_apply")
            dgamma, dbeta = link.dgamma, link.dbeta
            link.dz = link.sums = None
            ws = torch.empty(ws_floats, dtype=torch.float32, device=dev)
            N.check(lib.drc_bn_bwd(dy.data_ptr(), None, None, xs.data_ptr(), gamma_s.data_ptr(), None, mean_s.data_ptr(),
                                   invstd_s.data_ptr(), dxs.data_ptr(), None, dgamma_s.data_ptr(), dbeta_s.data_ptr(), ws.data_ptr(),
                                   sums.data_ptr(), _counter(dev)[8:].data_ptr(), M, c, MASK_NONE, _sms(dev), stream), "bn_bwd")
        else:
            ws = torch.empty(ws_floats // 2 * 3, dtype=torch.float32, device=dev)      # three accumulator rows per CTA
            N.check(lib.drc_bn_bwd_dual(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), xs.data_ptr(), gamma.data_ptr(),
                                        mean.data_ptr(), invstd.data_ptr(), gamma_s.data_ptr(), mean_s.data_ptr(), invstd_s.data_ptr(),
                                        dx.data_ptr(), dxs.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), dgamma_s.data_ptr(),
                                        dbeta_s.data_ptr(), ws.data_ptr(), sums.data_ptr(), sums[2 * c:].data_ptr(),
                                        _counter(dev)[8:].data_ptr(), M, c, _sms(dev), stream), "bn_bwd_dual")
        return dx, dxs, dgamma, dbeta, dgamma_s, dbeta_s, None, None, None, None, None


class FusedBatchNorm2d(nn.BatchNorm2d):
    """``nn.BatchNorm2d`` + optional fused residual add and ReLU.  When the producing ``ops.conv.Conv2d`` was called with
    ``bn=self`` its epilogue already computed this layer's batch statistics (``pending_stats``) and only the apply kernel runs."""

    def __init__(self, num_features: int, eps: float = 1e-5, momentum: float = 0.1, relu: bool = False):
        super().__init__(num_features, eps=eps, momentum=momentum)
        self.fuse_relu = relu
        self.pending_stats = None

    def _fused_ok(self, x: torch.Tensor) -> bool:
        return self.weight.dtype == torch.float32 and self.track_running_stats and fused_supported(x, self.training)

    def stat_request(self, x_in: torch.Tensor, channels: int):
        """Called by the producing convolution: a BnStatRequest if this layer will take the fused path for its output."""
        from .conv import BnStatRequest
        if not (self.training and self.weight.dtype == torch.float32 and self.track_running_stats and channels == self.num_features
                and channels <= 512 and os.environ.get("DRACO_BN", "fused") == "fused"
                and os.environ.get("DRACO_BN_STATS", "conv") == "conv" and bool(_lib().drc_bn_supported(channels))):
            return None
        upd = UPDATE_RUNNING_STATS
        return BnStatRequest(self.eps, self.momentum if self.momentum is not None else 0.1,
                             self.running_mean if upd else None, self.running_var if upd else None)

    def _count_batch(self) -> None:
        backend_counters["fused"] += 1
        if UPDATE_RUNNING_STATS and self.num_batches_tracked is not None:
            if _defer_counts:
                _pending_counts.append(self.num_batches_tracked)
            else:
                self.num_batches_tracked.add_(1)

    def _pair_ok(self, x: torch.Tensor, bn_s: "FusedBatchNorm2d", xs: torch.Tensor, relu: bool) -> bool:
        """Both layers on the fused path with their statistics from their convolutions' epilogues."""
        pend, pend_s = self.pending_stats, getattr(bn_s, "pending_stats", None)
        return (relu and isinstance(bn_s, FusedBatchNorm2d) and xs.shape == x.shape and xs.dtype == x.dtype
                and pend is not None and pend[0] is x and pend_s is not None and pend_s[0] is xs
                and self._fused_ok(x) and bn_s._fused_ok(xs))

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None, relu: Optional[bool] = None,
                residual_bn=None) -> torch.Tensor:
        """``residual_bn=(bn_s, xs)``: the residual is ``bn_s(xs)`` -- a downsampling block's projection shortcut.  When both
        layers take the fused path with convolution-epilogue statistics the pair runs as one op (``_BnPairFn``); otherwise this
        is ``self(x, residual=bn_s(xs))``."""
        relu = self.fuse_relu if relu is None else relu
        if residual_bn is not None:
            assert residual is None
            bn_s, xs = residual_bn
            if self._pair_ok(x, bn_s, xs, relu):
                (_, mean, invstd), self.pending_stats = self.pending_stats, None
                (_, mean_s, invstd_s), bn_s.pending_stats = bn_s.pending_stats, None
                bn_s._count_batch()
                self._count_batch()
                backend_counters["conv_stats"] = backend_counters.get("conv_stats", 0) + 2
                box = [None] if x.requires_grad else None
                y = _BnPairFn.apply(x, xs, self.weight, self.bias, bn_s.weight, bn_s.bias, mean, invstd, mean_s, invstd_s, box)
                if box is not None and box[0] is not None:
                    y._draco_bn_link = box[0]
                return y
            residual = bn_s(xs)
        pend, self.pending_stats = self.pending_stats, None
        if self._fused_ok(x) and (residual is None or residual.shape == x.shape):
            self._count_batch()
            upd = UPDATE_RUNNING_STATS
            mean = invstd = None
            if pend is not None and pend[0] is x:
                mean, invstd = pend[1], pend[2]                   # running statistics were updated by the convolution
                backend_counters["conv_stats"] = backend_counters.get("conv_stats", 0) + 1
            box = [None] if x.requires_grad else None
            y = _BnActFn.apply(x, residual, self.weight, self.bias, self.running_mean if upd else None,
                               self.running_var if upd else None, self.eps,
                               self.momentum if self.momentum is not None else 0.1, relu, mean, invstd, box)
            if box is not None and box[0] is not None:
                y._draco_bn_link = box[0]              # picked up by the ops.conv.Conv2d that consumes y (BatchNorm backward in its dgrad)
            return y
        assert pend is None, "a convolution produced fused statistics for a BatchNorm call that cannot use them"
        backend_counters["aten"] += 1
        if self.training and not UPDATE_RUNNING_STATS:
            y = F.batch_norm(x, None, None, self.weight, self.bias, True, 0.0, self.eps)
        else:
            y = super().forward(x)
        if residual is not None:
            y = y + residual
        return F.relu(y) if relu else y
