"""Convolution layer served by this repository's sm_90a kernels (see ``Conv2d``): wgmma tap-table / halo-reuse implicit GEMM
for 3x3 and 1x1 convolutions with stride 1 or 2 (fprop, dgrad, split-K wgrad; csrc/cuda/conv_tap_wgmma.cu,
conv_halo_wgmma.cu), the wgmma GEMM for the remaining pointwise layers (csrc/cuda/gemm_wgmma.cu) and CUDA-core kernels
for the 3-channel stem (csrc/cuda/conv_stem.cu).  In NHWC a 1x1 convolution *is* a GEMM:
``y[N*H*W, Cout] = x[N*H*W, Cin] @ W[Cout, Cin]^T`` -- both operands K-major, no im2col, no layout change (weights live in the
arena as ``[Cout, kH, kW, Cin]``).  The convolution epilogue can also produce the BatchNorm statistics of its output
(``BnStatRequest``).  ``backend_counters`` records which path served each call; ``DRACO_CONV=cudnn`` forces the library.

Reference counterpart: ``nn.Conv2d`` inside src/model_ops/resnet.py:14-64 / vgg.py:46-59 (PyTorch-0.3 CPU THNN).
"""
from __future__ import annotations

import os

import torch
from torch import nn

backend_counters = {"tcgen05": 0, "cudnn": 0}

# Weight gradients on a SIDE STREAM: dW of a layer is needed only when its bucket is pushed, while dX feeds the rest of the backward
# chain.  With this switch on, every wgrad kernel (+ its split-K fold) is enqueued on a side stream forked from the backward stream
# after dy / x are ready; the chain (BatchNorm backward -> dgrad -> ...) continues on the backward stream and overlaps with it (the
# BatchNorm kernels need no shared memory, so they co-reside with a convolution CTA on the same SM).  Consumers join explicitly:
# ``join_wgrad_stream()`` makes the CURRENT stream (or ``waiter``) wait for every wgrad enqueued so far -- the transport calls it
# before pushing a bucket, the worker after backward.  Set by the engine for processes that host ONE worker (a GPU that already
# runs several workers concurrently has nothing to gain).  Same kernels, same order per tensor: bit-identical results.
# Requires gradients that are STOLEN by autograd (p.grad is None before backward, the zero-copy mode of the worker): an
# accumulation ``p.grad += dw`` would run on the backward stream without waiting for the side stream.
WGRAD_SIDE_STREAM = False
_side_streams = {}
_side_pending = set()        # keys whose side stream holds work the backward stream has not joined yet
_side_keep = {}              # key -> tensors the side stream still reads (dy, x): kept alive until the forking stream has joined, so
                             # that the caching allocator cannot hand their memory to a later kernel of the forking stream while a
                             # weight-gradient kernel is still reading it (inside a CUDA-graph capture record_stream() does not help)


def _wgrad_stream(device) -> "torch.cuda.Stream":
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    if key not in _side_streams:
        _side_streams[key] = torch.cuda.Stream(device=device)
    _side_pending.add(key)
    return _side_streams[key]


def join_wgrad_stream(device, waiter: "torch.cuda.Stream" = None) -> None:
    """``waiter`` (default: the current stream) waits for every weight-gradient kernel forked from the current stream so far.
    A join by the forking stream itself settles the fork (later joins are no-ops until the next wgrad is forked -- which also keeps
    a CUDA-graph capture from depending on side-stream work enqueued before the capture began)."""
    cur = torch.cuda.current_stream(device)
    key = (device, cur.cuda_stream)
    if key not in _side_pending:
        return
    (waiter or cur).wait_stream(_side_streams[key])
    if waiter is None or waiter.cuda_stream == cur.cuda_stream:
        _side_pending.discard(key)
        _side_keep.pop(key, None)                  # the forking stream is ordered after every wgrad: their inputs may be reused


class _Conv1x1Fn(torch.autograd.Function):
    """x2: [M, Cin] (NHWC rows), w2: [Cout, Cin] -> y2: [M, Cout]."""

    @staticmethod
    def forward(ctx, x2, w2, bias):
        from . import kernels as K
        ctx.save_for_backward(x2, w2)
        ctx.has_bias = bias is not None
        return K.gemm_bf16(x2, w2, bias=bias)

    @staticmethod
    def backward(ctx, dy2):
        from . import kernels as K
        x2, w2 = ctx.saved_tensors
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dx = K.gemm_bf16(dy2, w2, b_mn=True) if ctx.needs_input_grad[0] else None
        dw = K.gemm_bf16(dy2, x2, a_mn=True, b_mn=True) if ctx.needs_input_grad[1] else None
        db = dy2.sum(0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return dx, dw, db


def _lib():
    import ctypes as C
    from .. import _native as N
    lib = N.cuda()
    if not getattr(lib, "_conv_ready", False):
        lib.drc_convg_supported.argtypes = [C.c_int] * 6
        lib.drc_convg_supported.restype = C.c_int
        lib.drc_convg_stat_slots.argtypes = [C.c_int] * 6
        lib.drc_convg_stat_slots.restype = C.c_int
        lib.drc_convg_plan.argtypes = [C.c_int] * 9 + [C.POINTER(C.c_int)]
        lib.drc_convg_plan.restype = C.c_int
        lib.drc_convg.argtypes = ([N.ptr, N.ptr, N.ptr] + [C.c_int] * 8 + [N.ptr, N.ptr, N.ptr, C.c_int] + [N.ptr] * 6
                                  + [C.c_float, C.c_float] + [N.ptr] * 7 + [C.c_int, C.c_int, N.ptr])
        lib.drc_convg.restype = C.c_int
        lib.drc_convg_wgrad_supported.argtypes = [C.c_int] * 6
        lib.drc_convg_wgrad_supported.restype = C.c_int
        lib.drc_convg_wgrad_plan.argtypes = [C.c_int] * 8 + [C.POINTER(C.c_longlong)]
        lib.drc_convg_wgrad_plan.restype = C.c_int
        lib.drc_convg_wgrad.argtypes = [N.ptr] * 4 + [C.c_int] * 9 + [N.ptr]
        lib.drc_convg_wgrad.restype = C.c_int
        lib.drc_conv_halo_supported.argtypes = [C.c_int] * 4
        lib.drc_conv_halo_supported.restype = C.c_int
        lib.drc_conv_halo_stat_slots.argtypes = [C.c_int] * 4
        lib.drc_conv_halo_stat_slots.restype = C.c_int
        lib.drc_conv_halo.argtypes = ([N.ptr, N.ptr, N.ptr] + [C.c_int] * 4 + [N.ptr, N.ptr, N.ptr] + [N.ptr] * 6
                                      + [C.c_float, C.c_float] + [N.ptr] * 7 + [C.c_int, C.c_int, N.ptr])
        lib.drc_conv_halo.restype = C.c_int
        lib.drc_conv_halo_wgrad.argtypes = [N.ptr] * 4 + [C.c_int] * 5 + [N.ptr]
        lib.drc_conv_halo_wgrad.restype = C.c_int
        lib.drc_conv_stem_supported.argtypes = [C.c_int] * 4
        lib.drc_conv_stem_supported.restype = C.c_int
        lib.drc_conv_stem_wgrad_parts.argtypes = [C.c_int] * 4
        lib.drc_conv_stem_wgrad_parts.restype = C.c_int
        lib.drc_conv_stem_fprop.argtypes = [N.ptr] * 4 + [C.c_int] * 3 + [N.ptr] * 6 + [C.c_float, C.c_float, C.c_int, C.c_int, N.ptr]
        lib.drc_conv_stem_fprop.restype = C.c_int
        lib.drc_conv_stem_wgrad.argtypes = [N.ptr] * 4 + [C.c_int] * 5 + [N.ptr]
        lib.drc_conv_stem_wgrad.restype = C.c_int
        lib._conv_ready = True
    return lib


class BnStatRequest:
    """Asks a convolution to produce the training-mode BatchNorm statistics of its output in its epilogue
    (csrc/cuda/conv_epilogue.cuh).  ``running_mean`` / ``running_var`` (may be None) receive the momentum update there as well;
    ``mean`` / ``invstd`` are filled by the call and handed to ``ops.norm`` (which then only runs its apply kernel)."""

    def __init__(self, eps: float, momentum: float, running_mean=None, running_var=None):
        self.eps, self.momentum = float(eps), float(momentum)
        self.running_mean, self.running_var = running_mean, running_var
        self.mean = self.invstd = None


def _stat_args(req, cout: int, slots: int, device):
    """(partial, counter, mean, invstd, running_mean, running_var, eps, momentum) for the C ABI."""
    if req is None:
        return (None, None, None, None, None, None, 0.0, 0.0), ()
    from .norm import _counter
    partial = torch.empty(slots * 2 * cout, dtype=torch.float32, device=device)
    req.mean = torch.empty(cout, dtype=torch.float32, device=device)
    req.invstd = torch.empty(cout, dtype=torch.float32, device=device)
    rm = req.running_mean.data_ptr() if req.running_mean is not None else None
    rv = req.running_var.data_ptr() if req.running_var is not None else None
    return ((partial.data_ptr(), _counter(device)[16:].data_ptr(), req.mean.data_ptr(), req.invstd.data_ptr(), rm, rv, req.eps,
             req.momentum), (partial,))


class BnBwdLink:
    """Connects a fused BatchNorm(+ReLU) layer with the convolution that consumes its output, for the backward pass: the
    convolution's dgrad epilogue masks its output with ``y > 0`` and reduces ``sum(dz)`` / ``sum(dz * xhat)`` per channel
    (csrc/cuda/conv_epilogue.cuh, BatchNorm-backward mode), so the BatchNorm's backward only runs its apply kernel.
    Created by ``ops.norm._BnActFn.forward`` (x, mean, invstd, relu), attached to the output tensor, picked up by
    ``Conv2d.forward``; the dgrad fills ``dz`` / ``sums`` / ``dgamma`` / ``dbeta``.  Valid when that convolution (and its
    ``fork``) is the only consumer of the BatchNorm output -- otherwise autograd hands the BatchNorm a different tensor than
    ``dz`` and it falls back to its own reduction."""
    __slots__ = ("x", "mean", "invstd", "relu", "dz", "sums", "dgamma", "dbeta")

    def __init__(self, x, mean, invstd, relu):
        self.x, self.mean, self.invstd, self.relu = x, mean, invstd, bool(relu)
        self.dz = self.sums = self.dgamma = self.dbeta = None


def _bwd_args(link, mask: torch.Tensor, c: int, slots: int, device):
    """C-ABI tail (bwd_x, bwd_mask, bwd_mean, bwd_invstd, bwd_sums, bwd_dgamma, bwd_dbeta) + statistics head for a dgrad that
    also reduces the BatchNorm backward of ``link``; without a link: null pointers."""
    if link is None:
        return (None,) * 7, None, ()
    from .norm import _counter
    partial = torch.empty(slots * 2 * c, dtype=torch.float32, device=device)
    link.sums = torch.empty(2 * c, dtype=torch.float32, device=device)
    link.dgamma = torch.empty(c, dtype=torch.float32, device=device)
    link.dbeta = torch.empty(c, dtype=torch.float32, device=device)
    head = (partial.data_ptr(), _counter(device)[16:].data_ptr(), None, None, None, None, 0.0, 0.0)
    tail = (link.x.data_ptr(), mask.data_ptr() if link.relu else None, link.mean.data_ptr(), link.invstd.data_ptr(),
            link.sums.data_ptr(), link.dgamma.data_ptr(), link.dbeta.data_ptr())
    return tail, head, (partial,)


# ---------------------------------------------------------------------------------------------------------------------
# tap-table implicit-GEMM kernels (csrc/cuda/conv_tap_wgmma.cu): stride 1 or 2, 1x1 or 3x3, fprop / dgrad / split-K wgrad
# ---------------------------------------------------------------------------------------------------------------------
def convg_tcgen05(act: torch.Tensor, weight: torch.Tensor, in_hw, stride: int, dgrad: bool = False,
                  bias: torch.Tensor = None, bn_stats: "BnStatRequest" = None, residual: torch.Tensor = None,
                  bn_bwd=None) -> torch.Tensor:
    """``dgrad=False``: ``act`` = x [N, Cin, H, W] -> y [N, Cout, H/stride, W/stride];  ``dgrad=True``: ``act`` = dy -> dx.
    ``in_hw`` is the spatial size of the forward input x; ``weight`` [Cout, Cin, ks, ks] in channels-last storage.
    ``residual``: channels-last bf16 tensor of the output's shape added in the epilogue (not for the 1x1 / stride-2 dgrad).
    ``bn_bwd`` = (BnBwdLink, y): stride-1 dgrad only -- the output is additionally masked with ``y > 0`` (y = the forward input of
    this convolution = the linked BatchNorm's output) and the BatchNorm-backward sums are left on the link."""
    from .. import _native as N
    from . import kernels as K
    lib = _lib()
    n = act.shape[0]
    h, w = in_hw
    cout, cin, ks = weight.shape[0], weight.shape[1], weight.shape[2]
    assert act.is_contiguous(memory_format=torch.channels_last)
    assert weight.permute(0, 2, 3, 1).is_contiguous(), "weights must be stored [Cout, ks, ks, Cin]"
    oshape = (n, cin, h, w) if dgrad else (n, cout, h // stride, w // stride)
    out = torch.empty(oshape, dtype=torch.bfloat16, device=act.device, memory_format=torch.channels_last)
    bf32 = bias.data_ptr() if bias is not None and bias.dtype == torch.float32 else None
    bb16 = bias.data_ptr() if bias is not None and bias.dtype == torch.bfloat16 else None
    sms = K.sm_count(act.device)
    tma = 0 if os.environ.get("DRACO_CONV_EPI", "tma") == "direct" else 1
    assert bn_stats is None or (tma and not dgrad)
    assert residual is None or (residual.shape == out.shape and residual.dtype == torch.bfloat16
                                and residual.is_contiguous(memory_format=torch.channels_last))
    slots = lib.drc_convg_stat_slots(n, h, w, cout, stride, sms) if (bn_stats is not None or bn_bwd is not None) else 0
    st, keep = _stat_args(bn_stats, cout, slots, act.device)
    tail, head, keep2 = _bwd_args(bn_bwd[0], bn_bwd[1], cin, slots, act.device) if bn_bwd is not None else ((None,) * 7, None, ())
    if bn_bwd is not None:
        assert dgrad and stride == 1 and tma and bn_stats is None and bn_bwd[0].x.shape == out.shape
        st = head
    N.check(lib.drc_convg(act.data_ptr(), weight.data_ptr(), out.data_ptr(), n, h, w, cin, cout, ks, stride, int(dgrad), bf32, bb16,
                          residual.data_ptr() if residual is not None else None, tma, *st, *tail, sms, act.device.index,
                          torch.cuda.current_stream().cuda_stream), "convg")
    del keep, keep2
    if bn_bwd is not None:
        bn_bwd[0].dz = out
    return out


def convg_plan(n: int, h: int, w: int, cin: int, cout: int, ks: int, stride: int, dgrad: int, num_sms: int = 132):
    """[block_n, cm, cn, grid, mode] the tap-convolution launcher picks for this layer (mode 0 = one CTA per tile, 1 = multicast
    cluster); host-side planning only, no GPU needed.  ``num_sms`` defaults to an H100 SXM."""
    import ctypes as C
    out = (C.c_int * 5)()
    if _lib().drc_convg_plan(n, h, w, cin, cout, ks, stride, int(dgrad), num_sms, out) != 0:
        return None
    return list(out)


def convg_wgrad_tcgen05(dy: torch.Tensor, x: torch.Tensor, ks: int, stride: int) -> torch.Tensor:
    """Weight gradient [Cout, Cin, ks, ks] (channels-last storage) of the strided / 1x1 / 3x3 convolution."""
    import ctypes as C
    from .. import _native as N
    from . import kernels as K
    lib = _lib()
    n, cout = dy.shape[0], dy.shape[1]
    cin, h, w = x.shape[1], x.shape[2], x.shape[3]
    assert dy.is_contiguous(memory_format=torch.channels_last) and x.is_contiguous(memory_format=torch.channels_last)
    sms = K.sm_count(dy.device)
    ws_elems = C.c_longlong(0)
    lib.drc_convg_wgrad_plan(n, h, w, cin, cout, ks, stride, sms, C.byref(ws_elems))
    ws = torch.empty(ws_elems.value, dtype=torch.float32, device=dy.device)
    dw = torch.empty((cout, ks, ks, cin), dtype=torch.bfloat16, device=dy.device).permute(0, 3, 1, 2)   # [Cout,Cin,ks,ks] view
    N.check(lib.drc_convg_wgrad(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), ws.data_ptr(), n, h, w, cin, cout, ks, stride, sms,
                                dy.device.index, torch.cuda.current_stream().cuda_stream), "convg_wgrad")
    return dw


def halo_supported(h: int, w: int, cin: int, cout: int) -> bool:
    """Halo-reuse kernel (csrc/cuda/conv_halo_wgmma.cu): 3x3 / stride 1, 64 -> 64 channels, H % 16 == 0, W % 8 == 0."""
    return os.environ.get("DRACO_CONV_HALO", "1") != "0" and bool(_lib().drc_conv_halo_supported(h, w, cin, cout))


def conv3x3_halo(act: torch.Tensor, weight: torch.Tensor, dgrad: bool = False, bias: torch.Tensor = None,
                 bn_stats: "BnStatRequest" = None, residual: torch.Tensor = None, bn_bwd=None) -> torch.Tensor:
    from .. import _native as N
    from . import kernels as K
    lib = _lib()
    n, _, h, w = act.shape
    assert act.is_contiguous(memory_format=torch.channels_last) and weight.permute(0, 2, 3, 1).is_contiguous()
    out = torch.empty((n, 64, h, w), dtype=torch.bfloat16, device=act.device, memory_format=torch.channels_last)
    bf32 = bias.data_ptr() if bias is not None and bias.dtype == torch.float32 else None
    bb16 = bias.data_ptr() if bias is not None and bias.dtype == torch.bfloat16 else None
    sms = K.sm_count(act.device)
    slots = lib.drc_conv_halo_stat_slots(n, h, w, sms) if (bn_stats is not None or bn_bwd is not None) else 0
    st, keep = _stat_args(bn_stats, 64, slots, act.device)
    tail, head, keep2 = _bwd_args(bn_bwd[0], bn_bwd[1], 64, slots, act.device) if bn_bwd is not None else ((None,) * 7, None, ())
    if bn_bwd is not None:
        assert dgrad and bn_stats is None and bn_bwd[0].x.shape == out.shape
        st = head
    assert residual is None or (residual.shape == out.shape and residual.dtype == torch.bfloat16
                                and residual.is_contiguous(memory_format=torch.channels_last))
    N.check(lib.drc_conv_halo(act.data_ptr(), weight.data_ptr(), out.data_ptr(), n, h, w, int(dgrad), bf32, bb16,
                              residual.data_ptr() if residual is not None else None, *st, *tail, sms,
                              act.device.index, torch.cuda.current_stream().cuda_stream), "conv_halo")
    del keep, keep2
    if bn_bwd is not None:
        bn_bwd[0].dz = out
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 3-channel stem (csrc/cuda/conv_stem.cu), CUDA cores.
# ---------------------------------------------------------------------------------------------------------------------
def conv_stem_fprop(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor = None, bn_stats: "BnStatRequest" = None) -> torch.Tensor:
    """x: channels-last bf16 [N, 3, H, W]; weight [64, 3, 3, 3] stored [Cout, 3, 3, Cin] -> y channels-last [N, 64, H, W]."""
    from .. import _native as N
    from . import kernels as K
    lib = _lib()
    n, _, h, w = x.shape
    assert x.is_contiguous(memory_format=torch.channels_last) and weight.permute(0, 2, 3, 1).is_contiguous()
    y = torch.empty((n, 64, h, w), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    b = bias.float().contiguous() if bias is not None else None
    sms = K.sm_count(x.device)
    st, keep = _stat_args(bn_stats, 64, lib.drc_conv_stem_wgrad_parts(n, h, w, sms) if bn_stats is not None else 0, x.device)
    N.check(lib.drc_conv_stem_fprop(x.data_ptr(), weight.data_ptr(), y.data_ptr(), b.data_ptr() if b is not None else None, n, h, w,
                                    *st, sms, x.device.index, torch.cuda.current_stream().cuda_stream), "conv_stem_fprop")
    del keep
    return y


def conv_stem_wgrad(dy: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    from .. import _native as N
    from . import kernels as K
    lib = _lib()
    n, _, h, w = x.shape
    assert dy.is_contiguous(memory_format=torch.channels_last) and x.is_contiguous(memory_format=torch.channels_last)
    sms = K.sm_count(dy.device)
    parts = lib.drc_conv_stem_wgrad_parts(n, h, w, sms)
    ws = torch.empty(parts * 64 * 27, dtype=torch.float32, device=dy.device)
    dw = torch.empty((64, 3, 3, 3), dtype=torch.bfloat16, device=dy.device).permute(0, 3, 1, 2)       # [Cout,Cin,3,3] view
    N.check(lib.drc_conv_stem_wgrad(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), ws.data_ptr(), n, h, w, sms, dy.device.index,
                                    torch.cuda.current_stream().cuda_stream), "conv_stem_wgrad")
    return dw


def conv3x3_halo_wgrad(dy: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """Weight gradient [64, 64, 3, 3] (stored [Cout, 3, 3, Cin]) of the 64 -> 64 3x3 / stride-1 layers: all nine taps from one resident
    halo per 128-pixel tile (csrc/cuda/conv_halo_wgmma.cu: wgrad_halo_wgmma_kernel)."""
    from .. import _native as N
    from . import kernels as K
    lib = _lib()
    n, _, h, w = x.shape
    assert dy.is_contiguous(memory_format=torch.channels_last) and x.is_contiguous(memory_format=torch.channels_last)
    sms = K.sm_count(dy.device)
    ws = torch.empty(lib.drc_conv_halo_stat_slots(n, h, w, sms) * 64 * 9 * 64, dtype=torch.float32, device=dy.device)
    dw = torch.empty((64, 3, 3, 64), dtype=torch.bfloat16, device=dy.device).permute(0, 3, 1, 2)
    N.check(lib.drc_conv_halo_wgrad(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), ws.data_ptr(), n, h, w, sms, dy.device.index,
                                    torch.cuda.current_stream().cuda_stream), "conv_halo_wgrad")
    return dw


class _ConvStemFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, bn_req):
        ctx.save_for_backward(x)
        ctx.has_bias = bias is not None
        ctx.set_materialize_grads(False)          # no zero-filled "gradients" for the statistics outputs
        y = conv_stem_fprop(x, weight, bias, bn_req)
        if bn_req is not None:
            mean, invstd = bn_req.mean, bn_req.invstd
        else:
            mean, invstd = x.new_empty(0, dtype=torch.float32), x.new_empty(0, dtype=torch.float32)
        ctx.mark_non_differentiable(mean, invstd)
        return y, mean, invstd

    @staticmethod
    def backward(ctx, dy, _dmean, _dinvstd):
        (x,) = ctx.saved_tensors
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        assert not ctx.needs_input_grad[0], "the stem kernel has no dgrad (network inputs carry no gradient)"
        dw = conv_stem_wgrad(dy, x) if ctx.needs_input_grad[1] else None
        db = dy.sum((0, 2, 3)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return None, dw, db, None


class _ConvGFn(torch.autograd.Function):
    """3x3 / 1x1, stride 1 / 2 convolution on the wgmma kernels.  Returns (y, mean, invstd, x_fork); mean / invstd are the
    fused BatchNorm statistics when ``bn_req`` is given (empty tensors otherwise) and carry no gradient.  ``x_fork`` (``fork=True``)
    is x again, for the OTHER consumer of x (the residual shortcut): its gradient comes back into this function and is added to dx
    inside the dgrad kernel's epilogue instead of by a separate elementwise kernel of autograd."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, bn_req, fork=False, in_link=None):
        ctx.save_for_backward(x, weight)
        # the BatchNorm(+ReLU) layer whose output x is: its backward reduction rides on this layer's dgrad epilogue (stride 1,
        # TMA-store epilogue, <= 512 channels)
        ctx.in_link = in_link if (in_link is not None and stride == 1 and weight.shape[1] <= 512
                                  and os.environ.get("DRACO_CONV_EPI", "tma") != "direct"
                                  and os.environ.get("DRACO_BN_BWD_FUSE", "0") == "1" and in_link.x.shape == x.shape) else None
        # OPT-IN: the fused epilogue adds row-offset integer divisions and exposed loads of y / x to every tile, against the one
        # reduce kernel it removes; it is not the default
        ctx.stride, ctx.has_bias = stride, bias is not None
        ctx.set_materialize_grads(False)          # no zero-filled "gradients" for the statistics outputs
        h, w = x.shape[2], x.shape[3]
        cout, cin, ks = weight.shape[0], weight.shape[1], weight.shape[2]
        ctx.halo = ks == 3 and stride == 1 and halo_supported(h, w, cin, cout)
        if ctx.halo:
            y = conv3x3_halo(x, weight, False, bias, bn_req)
        else:
            y = convg_tcgen05(x, weight, (h, w), stride, False, bias, bn_req)
        if bn_req is not None:
            mean, invstd = bn_req.mean, bn_req.invstd
        else:
            mean, invstd = x.new_empty(0, dtype=torch.float32), x.new_empty(0, dtype=torch.float32)
        ctx.mark_non_differentiable(mean, invstd)
        return y, mean, invstd, (x.view_as(x) if fork else x.new_empty(0))

    @staticmethod
    def backward(ctx, dy, _dmean, _dinvstd, dfork):
        x, weight = ctx.saved_tensors
        if dy is None:                                # only the fork branch carried a gradient
            return dfork, None, None, None, None, None, None
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        if dfork is not None and dfork.numel() == 0:
            dfork = None
        if dfork is not None and not (dfork.dtype == torch.bfloat16 and dfork.is_contiguous(memory_format=torch.channels_last)):
            dfork = dfork.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        fuse_fork = dfork is not None and ctx.needs_input_grad[0] and not (weight.shape[2] == 1 and ctx.stride > 1)
        dx = dw = db = None
        backend_counters["tcgen05"] += 1
        def wgrad():
            if ctx.halo and os.environ.get("DRACO_WGRAD_HALO", "1") != "0":
                return conv3x3_halo_wgrad(dy, x)
            return convg_wgrad_tcgen05(dy, x, weight.shape[2], ctx.stride)

        if ctx.needs_input_grad[1] and WGRAD_SIDE_STREAM:
            side = _wgrad_stream(dy.device)
            side.wait_stream(torch.cuda.current_stream(dy.device))          # dy and x are complete
            cur = torch.cuda.current_stream(dy.device)
            with torch.cuda.stream(side):
                dw = wgrad()
            _side_keep.setdefault((dy.device, cur.cuda_stream), []).extend((dy, x))     # alive until join_wgrad_stream()
            if not torch.cuda.is_current_stream_capturing():
                dw.record_stream(cur)              # allocated on the side stream, consumed (and later freed) by the backward stream
        if ctx.needs_input_grad[0]:
            res = dfork if fuse_fork else None
            link = ctx.in_link if (dfork is None or fuse_fork) else None       # the mask has to see the complete gradient of x
            bb = (link, x) if link is not None else None
            if ctx.halo:
                dx = conv3x3_halo(dy, weight, True, None, None, res, bb)
            else:
                dx = convg_tcgen05(dy, weight, x.shape[2:], ctx.stride, True, None, None, res, bb)
            if dfork is not None and not fuse_fork:
                dx = dx + dfork
        if ctx.needs_input_grad[1] and dw is None:
            dw = wgrad()
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum((0, 2, 3))
        return dx, dw, db, None, None, None, None


class Conv2d(nn.Conv2d):
    """``nn.Conv2d`` (same parameters / state_dict) whose CUDA bf16 channels-last forms run on this repository's kernels:

    * 3x3 and 1x1, stride 1 or 2, channel counts that are multiples of 64 -> tap-table / halo-reuse wgmma implicit GEMM;
    * 1x1 / stride 1 with other channel counts (multiples of 8, >= 64) -> the wgmma GEMM on NHWC rows;
    * the 3-channel 3x3 stem -> CUDA-core kernels of conv_stem.cu;
    * everything else (CPU, fp32, exotic geometry) -> ``nn.Conv2d`` (counted in ``backend_counters["cudnn"]``).

    ``forward(x, bn=module)`` additionally asks the kernel for the BatchNorm statistics of its output (see BnStatRequest) and
    leaves them on ``bn`` for the ``FusedBatchNorm2d`` call that follows.  ``DRACO_CONV=cudnn`` forces the library path."""

    def _common_ok(self, x: torch.Tensor) -> bool:
        return (os.environ.get("DRACO_CONV", "native") == "native" and self.dilation == (1, 1) and self.groups == 1 and x.is_cuda
                and x.dtype == torch.bfloat16 and self.weight.dtype == torch.bfloat16 and x.dim() == 4
                and x.is_contiguous(memory_format=torch.channels_last) and self.padding_mode == "zeros")

    def _pointwise_ok(self, x: torch.Tensor) -> bool:
        return (self._common_ok(x) and self.kernel_size == (1, 1) and self.stride == (1, 1) and self.padding == (0, 0)
                and self.in_channels % 8 == 0 and self.out_channels % 8 == 0 and self.in_channels >= 64 and self.out_channels >= 64)

    def _tap_ok(self, x: torch.Tensor) -> bool:
        ks, st = self.kernel_size[0], self.stride[0]
        if not (self._common_ok(x) and self.kernel_size in ((1, 1), (3, 3)) and self.stride in ((1, 1), (2, 2))
                and self.padding == (ks // 2, ks // 2) and self.weight.permute(0, 2, 3, 1).is_contiguous()):
            return False
        lib = _lib()
        h, w = x.shape[2], x.shape[3]
        return (bool(lib.drc_convg_supported(h, w, self.in_channels, self.out_channels, ks, st))
                and bool(lib.drc_convg_wgrad_supported(h, w, self.in_channels, self.out_channels, ks, st)))

    def _stem_ok(self, x: torch.Tensor) -> bool:
        return (self._common_ok(x) and self.kernel_size == (3, 3) and self.stride == (1, 1) and self.padding == (1, 1)
                and self.in_channels == 3 and self.out_channels == 64 and not x.requires_grad
                and self.weight.permute(0, 2, 3, 1).is_contiguous()
                and bool(_lib().drc_conv_stem_supported(x.shape[2], x.shape[3], 3, 64)))

    def forward(self, x: torch.Tensor, bn: nn.Module = None, fork: bool = False):
        """``fork=True`` returns ``(y, x_fork)``: ``x_fork`` is x for the second consumer of x (the shortcut branch of a residual
        block); on the native path the gradient that comes back through it is added inside this layer's dgrad epilogue."""
        if fork:
            if self._tap_ok(x) and x.requires_grad and os.environ.get("DRACO_CONV_FORK", "1") != "0":
                backend_counters["tcgen05"] += 1
                req = bn.stat_request(x, self.out_channels) if (bn is not None and hasattr(bn, "stat_request")) else None
                y, mean, invstd, xf = _ConvGFn.apply(x, self.weight, self.bias, self.stride[0], req, True,
                                                     getattr(x, "_draco_bn_link", None))
                if req is not None:
                    bn.pending_stats = (y, mean, invstd)
                return y, xf
            return self.forward(x, bn=bn), x
        if self._stem_ok(x):
            backend_counters["native_stem"] = backend_counters.get("native_stem", 0) + 1
            req = bn.stat_request(x, self.out_channels) if (bn is not None and hasattr(bn, "stat_request")) else None
            y, mean, invstd = _ConvStemFn.apply(x, self.weight, self.bias, req)
            if req is not None:
                bn.pending_stats = (y, mean, invstd)
            return y
        if self._tap_ok(x):
            backend_counters["tcgen05"] += 1
            req = bn.stat_request(x, self.out_channels) if (bn is not None and hasattr(bn, "stat_request")) else None
            y, mean, invstd, _ = _ConvGFn.apply(x, self.weight, self.bias, self.stride[0], req, False,
                                                getattr(x, "_draco_bn_link", None) if x.requires_grad else None)
            if req is not None:
                bn.pending_stats = (y, mean, invstd)
            return y
        if not self._pointwise_ok(x):
            backend_counters["cudnn"] += 1
            return super().forward(x)
        backend_counters["tcgen05"] += 1
        n, c, h, w = x.shape
        x2 = x.permute(0, 2, 3, 1).reshape(n * h * w, c)                    # view: NHWC rows
        w2 = self.weight.permute(0, 2, 3, 1).reshape(self.out_channels, c)  # view of the [Cout,1,1,Cin] arena storage
        if not w2.is_contiguous():
            w2 = w2.contiguous()
        y2 = _Conv1x1Fn.apply(x2, w2, self.bias)
        return y2.view(n, h, w, self.out_channels).permute(0, 3, 1, 2)      # channels-last [N, Cout, H, W]
