"""Linear layer backed by the hand-written wgmma GEMM (``csrc/cuda/gemm_wgmma.cu``).

All three products of a linear layer run on the same kernel without transpose copies, by describing operands to TMA
/ wgmma as K-major or MN-major:

    y  = x  W^T   A = x  (K-major)   B = W  (K-major)     + fused bias (+ReLU) epilogue
    dx = dy W     A = dy (K-major)   B = W  (MN-major)
    dW = dy^T x   A = dy (MN-major)  B = x  (MN-major)

Narrow heads (10 classes) are zero-padded to a multiple of 8 in the backward pass so that they stay on this kernel too; other
shapes whose rows are not 16-byte multiples and non-bf16 / CPU tensors take the cuBLAS / ATen path -- that is a per-call shape gate, not a silent global fallback: ``backend_counters`` records
which path served every call so tests and the bench can assert the tensor-core path ran.
"""
from __future__ import annotations

import math
import os

import torch
import torch.nn.functional as F
from torch import nn

backend_counters = {"tcgen05": 0, "aten": 0}


def _use_native(x: torch.Tensor) -> bool:
    return x.is_cuda and x.dtype == torch.bfloat16 and os.environ.get("DRACO_LINEAR", "tcgen05") == "tcgen05"


class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        from . import kernels as K
        # x is 2-d and contiguous (Linear.forward flattens outside the Function so the output is never a view)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        if K.gemm_supported(x, weight) and weight.is_contiguous():
            backend_counters["tcgen05"] += 1
            return K.gemm_bf16(x, weight, bias=bias)
        backend_counters["aten"] += 1
        return F.linear(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        from . import kernels as K
        x, weight = ctx.saved_tensors
        dy2 = dy if dy.is_contiguous() else dy.contiguous()
        x2 = x
        dx = dw = db = None
        nout = weight.shape[0]
        if nout % 8 and weight.shape[1] >= 64 and x2.shape[1] >= 64 and K.gemm_supported(x2, weight):
            # narrow heads (10 classes): a row of dy / a column block of W is not a 16-byte multiple, which TMA requires.  Pad the
            # class dimension with zeros to the next multiple of 8 (two tiny copies) and stay on the tensor-core kernel.
            pad = 8 - nout % 8
            from .pool import head_prep
            dy_p, db = head_prep(dy2, nout + pad, ctx.has_bias and ctx.needs_input_grad[2])     # pad + bias gradient, one launch
            if ctx.needs_input_grad[0]:
                backend_counters["tcgen05"] += 1
                dx = K.gemm_bf16(dy_p, F.pad(weight, (0, 0, 0, pad)), b_mn=True)
            if ctx.needs_input_grad[1]:
                backend_counters["tcgen05"] += 1
                dw = K.gemm_bf16(dy_p, x2, a_mn=True, b_mn=True)[:nout]
            return dx, dw, db
        if ctx.needs_input_grad[0]:
            if K.gemm_supported(dy2, weight) and weight.shape[1] >= 64:
                backend_counters["tcgen05"] += 1
                dx = K.gemm_bf16(dy2, weight, b_mn=True)
            else:
                backend_counters["aten"] += 1
                dx = dy2 @ weight
        if ctx.needs_input_grad[1]:
            if K.gemm_supported(dy2, x2) and x2.shape[1] >= 64:
                backend_counters["tcgen05"] += 1
                dw = K.gemm_bf16(dy2, x2, a_mn=True, b_mn=True)
            else:
                backend_counters["aten"] += 1
                dw = dy2.t() @ x2
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.sum(0)
        return dx, dw, db


class Linear(nn.Module):
    """Drop-in ``nn.Linear`` (same parameter names / init) whose CUDA bf16 path is the wgmma GEMM."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True) -> None:
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.empty(out_features)) if bias else None
        self.reset_parameters()

    def reset_parameters(self) -> None:
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1.0 / math.sqrt(self.in_features) if self.in_features > 0 else 0.0
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if _use_native(x) and self.weight.dtype == torch.bfloat16:
            x2 = x.reshape(-1, x.shape[-1])
            if not x2.is_contiguous():
                x2 = x2.contiguous()
            y = _LinearFn.apply(x2, self.weight, self.bias)
            return y if x.dim() == 2 else y.reshape(*x.shape[:-1], self.out_features)
        return F.linear(x, self.weight, self.bias)

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}"
