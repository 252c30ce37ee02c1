"""draco_b200: a Hopper-native (H100) Byzantine-resilient data-parallel trainer with Draco's capabilities.

Layout
  codes/     repetition + cyclic (Fourier) gradient codes, adversary model, fp64 oracles
  models/    LeNet, FC, ResNet-18..152, VGG-11..19 (+ *Split layer-wise backward drivers)
  ops/       launchers for the sm_90a kernels (push/encode, vote, decode, robust aggregators, wgmma GEMM)
  optim/     SGDModified / AdamModified (external-gradient optimizers)
  parallel/  arenas, symmetric memory, placement, PS / worker roles, fused (nvl) and collective (nccl/gloo) engines, Trainer
  data/      datasets + identical-batch plans
  utils/     codec, checkpoint, metrics
  cli/       distributed_nn / distributed_evaluator / single_machine / cluster launcher entry points
"""
from .config import JobConfig

__version__ = "0.1.0"
__all__ = ["JobConfig", "Trainer", "build_model"]


def __getattr__(name):
    if name == "Trainer":
        from .parallel.trainer import Trainer
        return Trainer
    if name == "build_model":
        from .models import build_model
        return build_model
    raise AttributeError(name)
