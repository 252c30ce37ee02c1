"""Cluster-shape sweep of the tap convolution (csrc/cuda/conv_tap_wgmma.cu): for the ResNet-18/CIFAR layers at B=128, time
fprop (with fused BatchNorm statistics) and dgrad for every cluster shape cm x cn and tile width the kernel supports
(DRACO_CONV_CLUSTER override), with the same CUDA-graph timing as tools/bench_conv.py, and check each variant against the
no-cluster result (bit-exact: same MMA order per tile).  Writes gpurun_out/conv_cluster_sweep.json; the planner
(plan_tap) is calibrated against this table."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from draco_b200.ops import conv as C  # noqa: E402

dev = torch.device("cuda", 0)
REP = 10


def timeit(fn, replays=8):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REP):
            fn()
    g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(replays):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return round(s.elapsed_time(e) / (replays * REP) * 1e3, 2)          # us per launch


def cl(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def wt(k, c, ks):
    return (torch.randn(k, c, ks, ks, device=dev) * 0.05).to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


N = 128
SHAPES = [(128, 128, 16, 3, 1), (256, 256, 8, 3, 1), (512, 512, 4, 3, 1), (64, 128, 32, 3, 2), (128, 256, 16, 3, 2),
          (256, 512, 8, 3, 2), (64, 128, 32, 1, 2), (256, 512, 8, 1, 2), (64, 64, 32, 3, 1)]
CONFIGS = os.environ["SWEEP_CONFIGS"].split(";") if os.environ.get("SWEEP_CONFIGS") else ["1,1,128", "1,1,64", "2,1,128", "4,1,128", "8,1,128", "1,2,128", "2,2,128", "4,2,128", "2,4,128", "1,2,64", "2,2,64",
           "4,2,64", "2,4,64", "1,4,64", "1,8,64", "4,1,64", "8,1,64", "auto"]
rows = []
for (c, k, hw, ks, st) in SHAPES:
    x = cl(torch.randn(N, c, hw, hw, device=dev))
    w = wt(k, c, ks)
    dy = cl(torch.randn(N, k, hw // st, hw // st, device=dev))
    req = C.BnStatRequest(1e-5, 0.1)
    os.environ["DRACO_CONV_CLUSTER"] = "1,1"
    ref_y, ref_dx = C.convg_tcgen05(x, w, (hw, hw), st), C.convg_tcgen05(dy, w, (hw, hw), st, True)
    for cfg in CONFIGS:
        os.environ["DRACO_CONV_CLUSTER"] = cfg                # "auto": the traffic model picks (default without the variable: 1,1)
        row = {"Cin": c, "Cout": k, "HW": hw, "ks": ks, "stride": st, "cfg": cfg}
        for name, dg in (("fprop", 0), ("dgrad", 1)):
            plan = C.convg_plan(N, hw, hw, c, k, ks, st, dg)
            want = None if cfg == "auto" else [int(v) for v in cfg.split(",")]
            if want is not None and [plan[1], plan[2], plan[0]] != want:
                row[name + "_us"] = None                      # shape not realisable for this layer
                continue
            row[name + "_plan"] = plan
            if dg:
                fn = lambda: C.convg_tcgen05(dy, w, (hw, hw), st, True)                    # noqa: E731
                got = fn()
                ok = torch.equal(got, ref_dx)
                row[name + "_maxdiff"] = float((got.float() - ref_dx.float()).abs().max())
            else:
                fn = lambda: C.convg_tcgen05(x, w, (hw, hw), st, False, None, req)          # noqa: E731
                got = fn()
                ok = torch.equal(got, ref_y)
                row[name + "_maxdiff"] = float((got.float() - ref_y.float()).abs().max())
            torch.cuda.synchronize()
            row[name + "_exact"] = bool(ok)
            row[name + "_us"] = timeit(fn)
        rows.append(row)
        print(json.dumps(row), flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open("gpurun_out/conv_cluster_sweep.json", "w"), indent=1)
