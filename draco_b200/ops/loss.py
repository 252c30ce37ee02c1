"""Classifier-head loss: softmax cross-entropy + Prec@1 / Prec@5, optionally as ONE sm_90a kernel.

``cross_entropy_with_metrics(logits, labels, metrics, scale)`` returns the mean loss (differentiable w.r.t. ``logits``) and
adds ``scale * (loss, prec1 %, prec5 %)`` to the 3-element ``metrics`` tensor.  Default path: the PyTorch ops the reference
uses (``F.cross_entropy`` + its ``accuracy`` helper, src/worker/utils.py:22-35).  With ``DRACO_FUSED_LOSS=1`` on CUDA the
whole tail -- including the gradient w.r.t. the logits -- is produced by ``csrc/cuda/loss_fused.cu`` in one launch
(~20 dependent launches otherwise); the backward pass is then a single scale by the incoming gradient.
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch
import torch.nn.functional as F


def accuracy(output: torch.Tensor, target: torch.Tensor, topk=(1, 5)) -> List[torch.Tensor]:
    """Prec@k in percent (the reference carries four copies of this helper, e.g. src/worker/utils.py:22-35)."""
    maxk = min(max(topk), output.shape[1])
    _, pred = output.float().topk(maxk, 1, True, True)
    correct = pred.t().eq(target.view(1, -1))
    return [correct[:min(k, maxk)].reshape(-1).float().sum() * (100.0 / target.shape[0]) for k in topk]


def _lib():
    import ctypes as C
    from .. import _native as N
    lib = N.cuda()
    if not getattr(lib, "_ce_ready", False):
        lib.drc_ce_fused.argtypes = [N.ptr, C.c_int, N.ptr, N.ptr, N.ptr, N.ptr, C.c_float, C.c_int, C.c_int, N.ptr]
        lib.drc_ce_fused.restype = C.c_int
        lib._ce_ready = True
    return lib


class _FusedCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, metrics, scale):
        from .. import _native as N
        assert logits.dim() == 2 and logits.is_contiguous() and logits.dtype in (torch.bfloat16, torch.float32)
        assert labels.dtype == torch.int64 and labels.is_contiguous()
        b, c = logits.shape
        dlogits = torch.empty_like(logits)
        loss = torch.empty(1, dtype=torch.float32, device=logits.device)
        N.check(_lib().drc_ce_fused(logits.data_ptr(), int(logits.dtype == torch.bfloat16), labels.data_ptr(), dlogits.data_ptr(),
                                    loss.data_ptr(), metrics.data_ptr() if metrics is not None else None, float(scale), b, c,
                                    torch.cuda.current_stream().cuda_stream), "ce_fused")
        ctx.save_for_backward(dlogits)
        return loss.view(())

    @staticmethod
    def backward(ctx, grad_out):
        (dlogits,) = ctx.saved_tensors
        return dlogits * grad_out.to(dlogits.dtype), None, None, None


def fused_enabled(logits: torch.Tensor) -> bool:
    return (os.environ.get("DRACO_FUSED_LOSS", "1") == "1" and logits.is_cuda and logits.dim() == 2
            and logits.dtype in (torch.bfloat16, torch.float32))


def cross_entropy_with_metrics(logits: torch.Tensor, labels: torch.Tensor, metrics: Optional[torch.Tensor] = None,
                               scale: float = 1.0) -> torch.Tensor:
    if fused_enabled(logits):
        return _FusedCE.apply(logits.contiguous(), labels, metrics, scale)
    loss = F.cross_entropy(logits.float(), labels)
    if metrics is not None:
        with torch.no_grad():
            p1, p5 = accuracy(logits.detach(), labels)
            metrics += torch.stack([loss.detach(), p1, p5]) * scale
    return loss
