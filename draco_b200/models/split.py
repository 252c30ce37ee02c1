"""Layer-wise ("split") backward drivers.

The reference's ``LeNetSplit`` / ``FC_NN_Split`` / ``ResNetSplit*`` detach every layer's input so that
backward can be driven one layer at a time and each layer's gradient shipped to the PS while the
remaining layers are still back-propagating (src/model_ops/resnet_split.py:431-623 ``backward_normal``,
:760-860 ``backward_coded``, :739-758 ``backward_single``; lenet.py:114-218; fc_nn.py:94-199) -- with MPI
calls, the adversary and the compressor living *inside the model*.

This design keeps the capability (gradients become visible to the transport in reverse layer order
while backward is still running, so the push overlaps backprop) but not the layering violation: a
``SplitBackwardMixin`` model exposes the same three drivers, implemented with autograd's
post-accumulate-grad hooks; what happens to a finished gradient is a callback supplied by the worker
runtime.  ``parallel/worker.py::WorkerCompute.forward_backward`` drives every backward pass through them:
``backward_normal(loss, on_ready)`` when the transport overlaps the push with backprop (the callback counts
down the bucket and enqueues the fused encode+push kernel on a side stream), ``backward_coded`` for the
earlier sub-batches of a cyclic-code worker, ``backward_single`` otherwise.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import torch

GradCallback = Callable[[int, torch.nn.Parameter], None]


class SplitBackwardMixin:
    """Adds ``backward_normal`` / ``backward_coded`` / ``backward_single`` to an ``nn.Module``."""

    def _split_params(self) -> List[torch.nn.Parameter]:
        return [p for p in self.parameters() if p.requires_grad]   # type: ignore[attr-defined]

    def _run_hooked(self, loss: torch.Tensor, on_ready: Optional[GradCallback]) -> List[torch.Tensor]:
        params = self._split_params()
        index = {id(p): i for i, p in enumerate(params)}
        order: List[int] = []
        handles = []
        for p in params:
            def hook(param, _index=index, _order=order):
                i = _index[id(param)]
                _order.append(i)
                if on_ready is not None:
                    on_ready(i, param)
            handles.append(p.register_post_accumulate_grad_hook(hook))
        try:
            loss.backward()
        finally:
            for h in handles:
                h.remove()
        self._last_ready_order = order
        return [p.grad for p in params]

    def backward_normal(self, loss: torch.Tensor, on_ready: Optional[GradCallback] = None) -> List[torch.Tensor]:
        """Send-as-you-go backward: ``on_ready(param_index, param)`` fires as soon as a parameter's
        gradient is final, in reverse layer order (reference: resnet_split.py:431-623)."""
        return self._run_hooked(loss, on_ready)

    def backward_coded(self, loss: torch.Tensor) -> List[torch.Tensor]:
        """Collect-then-send backward (reference: resnet_split.py:760-860): returns gradients in
        *reverse parameter order*, the order the reference's coded workers transmit them in."""
        grads = self._run_hooked(loss, None)
        return list(reversed(grads))

    def backward_single(self, loss: torch.Tensor) -> None:
        """Plain single-machine backward (reference: resnet_split.py:739-758)."""
        loss.backward()

    @property
    def ready_order(self) -> List[int]:
        """Parameter indices in the order their gradients became final during the last backward."""
        return list(getattr(self, "_last_ready_order", []))


def make_split(cls: type, name: str) -> type:
    """Create ``<Model>Split`` = model + split-backward drivers."""
    return type(name, (SplitBackwardMixin, cls), {"__doc__": f"{cls.__name__} with layer-wise backward drivers."})
