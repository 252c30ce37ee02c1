"""NVLink roofline sweep of the fused communication paths (encode / decode GB/s vs the NVLink roofline).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29510 tools/bench_push.py

Topology of the product: rank 0 = PS, ranks 1..N-1 = one worker each (with N = 1 or 2 the logical workers are packed).  For a
sweep of gradient sizes (default 1, 4, 16, 45, 94, 200 MB of fp32 -- 45 MB = ResNet-18, 94 MB = ResNet-50) the tool times, on the
device with CUDA events, each fused path IN ISOLATION (a process-group barrier separates the phases, max over ranks):

  push     : every worker's push_encode kernel (repetition encode + adversary hook + 16-byte peer stores into its PS slot) run
             concurrently -> per-worker GB/s (egress of one GPU, roofline 770 GB/s measured peer copy / 900 nominal) and PS
             ingress GB/s (P workers x bytes into one GPU: the same per-direction roofline)
  decode   : PS-side vote (compare + resolve) over the P slots: HBM-bound, reads P x bytes (roofline MEASURED_PEAKS hbm_gbs)
  update   : aggregate_update = select-sum + SGD-momentum + broadcast of the fresh parameters to every worker, once through the
             NVLS multicast mapping (one multimem.st stream: PS egress = bytes) and once through unicast peer stores (PS egress =
             (N-1) x bytes); roofline = egress bytes / 770 GB/s

Prints one JSON line per size on rank 0 and writes gpurun_out/push_sweep_N<N>.json.
"""
from __future__ import annotations

import json
import os
import sys

import torch
import torch.distributed as dist
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from draco_b200.codes.repetition import group_assign  # noqa: E402
from draco_b200.ops import kernels as K  # noqa: E402
from draco_b200.parallel.arena import ArenaLayout  # noqa: E402
from draco_b200.parallel.placement import Placement  # noqa: E402
from draco_b200.parallel.symm import SymmContext  # noqa: E402
from draco_b200.parallel.trainer import init_distributed  # noqa: E402

LINK_GBS = 450.0          # H100 SXM NVLink 4, data-sheet rate per direction (900 GB/s bidirectional); not a measured rate
FLAG_BYTES = 1 << 16
REPS = int(os.environ.get("PUSH_REPS", "10"))


class _Flat(nn.Module):
    def __init__(self, numel: int, ntensors: int = 16):
        super().__init__()
        per = max(1024, numel // ntensors // 1024 * 1024)
        self.ps = nn.ParameterList([nn.Parameter(torch.zeros(per)) for _ in range(ntensors)])


def main() -> int:
    rank, world, local = init_distributed("nvl")
    dev = torch.device("cuda", local % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    P = 7
    place = Placement(P, world)
    local_workers = place.local_workers(rank)
    sizes_mb = [float(x) for x in os.environ.get("PUSH_SIZES_MB", "1,4,16,45,94,200").split(",")]
    try:
        hbm = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        hbm = 6650.0
    rows = []

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    def timed(fn):
        """max over ranks of the mean device time (ms) of REPS back-to-back runs of fn (each separated by a group barrier)."""
        tot = 0.0
        for it in range(REPS + 2):
            barrier()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            if it >= 2:
                tot += s.elapsed_time(e)
        t = torch.tensor([tot / REPS], dtype=torch.float64, device=dev if world == 1 or dist.get_backend() != "gloo" else "cpu")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    for mb in sizes_mb:
        numel = int(mb * 1e6 / 4)
        layout = ArenaLayout.from_model(_Flat(numel), False, channels_last=False)
        D = layout.total
        nbytes = D * 4
        symm = SymmContext(dev, rank, world, None)
        regA = symm.alloc("params", nbytes + FLAG_BYTES, None)
        params = regA.tensor[:nbytes].view(torch.float32)
        if rank == 0:
            regB = symm.alloc("grad_in", P * nbytes + FLAG_BYTES)
            grad_in = regB.tensor[: P * nbytes].view(torch.float32)
        allp = list(range(world))
        mapA = symm.share("params", exporters=allp, importers=[0])
        mapB = symm.share("grad_in", exporters=[0], importers=allp)
        mc = symm.bind_multicast("params") if world > 1 else None
        step = torch.ones(1, dtype=torch.int64, device=dev)
        counters = torch.zeros(16, dtype=torch.int32, device=dev)
        # every group member pushes the same gradient (so the vote has real agreeing replicas to compare)
        groups = group_assign(P, 3)
        g32 = {w: [torch.randn(D, generator=torch.Generator().manual_seed(groups.rank_to_group[w]), dtype=torch.float32).to(dev)]
               for w in local_workers}

        def push():
            for w in local_workers:
                K.push_encode(layout, g32[w], [None], mapB[0].ptr + (w - 1) * nbytes, step_ptr=step, worker=w - 1,
                              done_counter=counters[w:w + 1], flag=None,
                              grid=int(os.environ.get("PUSH_CTAS", "16")) if rank != 0 or world == 1 else 2 * K.sm_count())

        t_push = timed(push) if local_workers or True else 0.0
        row = {"size_mb": round(nbytes / 1e6, 2), "n_gpus": world, "workers": P, "push_ms": t_push}
        per_worker = max(len(place.local_workers(p)) for p in range(world))
        row["push_gbs_per_gpu_egress"] = per_worker * nbytes / 1e6 / t_push
        remote = sum(len(place.local_workers(p)) for p in range(1, world))
        row["ps_ingress_gbs"] = remote * nbytes / 1e6 / t_push if remote else None
        row["push_frac_of_link"] = (max(row["push_gbs_per_gpu_egress"] if world > 1 else 0.0, row["ps_ingress_gbs"] or 0.0) / LINK_GBS) if world > 1 else None
        if world == 1:
            row["push_frac_of_hbm"] = 2 * P * nbytes / 1e6 / t_push / hbm          # local slot: read + write through HBM
        G = len(groups.groups)
        if rank == 0:
            table = torch.from_numpy(groups.as_table()).to(dev)
            T = layout.ntensors
            neq = torch.zeros(G, T, dtype=torch.int32, device=dev)
            win = torch.zeros(G, T, dtype=torch.int32, device=dev)
            mom = layout.new_arena(dev)
            from draco_b200 import JobConfig
            from draco_b200.parallel.ps import hyperparams_tensor
            hp = hyperparams_tensor(JobConfig(lr=0.01, momentum=0.9), dev)
            dst = [mapA[p].ptr for p in place.worker_procs() if p != 0]

        def decode():
            if rank == 0:
                K.vote(layout, grad_in, D, table, neq, win)

        def update(mcast):
            if rank == 0:
                K.aggregate_update(layout, grad_in, D, K=G, scale=1.0 / G, select=win, params=params, momentum=mom, hp=hp, step_ptr=step,
                                   done_counter=counters[0:1], mc_params=mc if mcast else None, dst=[] if (mcast and mc) else dst)

        t_dec = timed(decode)
        row["decode_ms"] = t_dec
        row["decode_gbs"] = P * nbytes / 1e6 / t_dec
        row["decode_frac_of_hbm"] = row["decode_gbs"] / hbm
        for name, mcast in (("multicast", True), ("unicast", False)):
            if mcast and not mc:
                row["update_multicast_ms"] = None
                continue
            t = timed(lambda: update(mcast))
            egress = nbytes * (1 if mcast else max(world - 1, 0))
            row[f"update_{name}_ms"] = t
            row[f"update_{name}_egress_gbs"] = egress / 1e6 / t if world > 1 else None
            row[f"update_{name}_frac_of_link"] = (egress / 1e6 / t / LINK_GBS) if world > 1 else None
            # HBM side of the same kernel: reads G winner rows + params + momentum, writes params + momentum (+ local copy)
            row[f"update_{name}_hbm_gbs"] = (G + 4) * nbytes / 1e6 / t
        barrier()
        if rank == 0:
            rows.append(row)
            print(json.dumps(row), flush=True)
        del g32, params
        if rank == 0:
            del grad_in
        symm.close()
        barrier()
    if rank == 0:
        os.makedirs("gpurun_out", exist_ok=True)
        json.dump(rows, open(f"gpurun_out/push_sweep_N{world}.json", "w"), indent=1)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
