"""ONE process, TWO GPUs: launch the fused communication kernels with their destination in the PEER GPU's memory, for an ncu capture
with NVLink byte counters (`ncu --section Nvlink_Topology --section Nvlink_Tables --metrics nvltx__bytes.sum,nvlrx__bytes.sum ...`).

  push_encode_kernel       on cuda:0, destination slot on cuda:1     -> NVLink TX bytes of GPU0 ~= gradient bytes (encode fused with the push)
  aggregate_update_kernel  on cuda:0, unicast destination on cuda:1  -> NVLink TX bytes ~= parameter bytes per destination
(The NVLS multicast variant needs the multi-process symmetric-memory context and is measured by tools/bench_push.py instead.)
Also times both kernels with CUDA events and prints achieved GB/s.
"""
import ctypes
import json
import os
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from draco_b200 import JobConfig  # noqa: E402
from draco_b200.ops import kernels as K  # noqa: E402
from draco_b200.parallel.arena import ArenaLayout  # noqa: E402
from draco_b200.parallel.ps import hyperparams_tensor  # noqa: E402


class _Flat(nn.Module):
    def __init__(self, numel, ntensors=16):
        super().__init__()
        self.ps = nn.ParameterList([nn.Parameter(torch.zeros(numel // ntensors // 1024 * 1024)) for _ in range(ntensors)])


def main():
    assert torch.cuda.device_count() >= 2
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)
    torch.cuda.set_device(d0)
    rt = ctypes.CDLL("libcudart.so")
    rc = rt.cudaDeviceEnablePeerAccess(1, 0)
    assert rc in (0, 704), rc                                   # 704: already enabled
    mb = float(os.environ.get("NVL_MB", "45"))
    layout = ArenaLayout.from_model(_Flat(int(mb * 1e6 / 4)), False, channels_last=False)
    D = layout.total
    grad = [torch.randn(D, device=d0)]
    slot_remote = torch.zeros(2, D, device=d1)                  # "PS" memory on the peer
    params_remote = torch.zeros(D, device=d1)
    step = torch.ones(1, dtype=torch.int64, device=d0)
    cnt = torch.zeros(8, dtype=torch.int32, device=d0)
    grad_in = torch.randn(2, D, device=d0)
    params, mom = torch.zeros(D, device=d0), torch.zeros(D, device=d0)
    hp = hyperparams_tensor(JobConfig(lr=0.01, momentum=0.9), d0)
    out = {}
    for name, fn, nbytes in (
            ("push_encode_16cta", lambda: K.push_encode(layout, grad, [None], slot_remote[0], step_ptr=step, worker=0, done_counter=cnt[0:1], grid=16), D * 4),
            ("push_encode_full_grid", lambda: K.push_encode(layout, grad, [None], slot_remote[1], step_ptr=step, worker=0, done_counter=cnt[1:2], grid=K.sm_count()), D * 4),
            ("aggregate_update_unicast", lambda: K.aggregate_update(layout, grad_in, D, K=2, scale=0.5, params=params, momentum=mom, hp=hp, step_ptr=step,
                                                                   done_counter=cnt[2:3], dst=[params_remote.data_ptr()]), D * 4)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(5):
            fn()
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / 5
        out[name] = {"ms": ms, "nvlink_gbs": nbytes / 1e6 / ms, "bytes": nbytes}
    torch.cuda.synchronize()
    assert torch.equal(slot_remote[0].cpu(), grad[0].cpu()) and torch.equal(params_remote.cpu(), params.cpu())
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
