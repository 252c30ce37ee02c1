"""Where do the microseconds of a tap-convolution launch go?  Per-CTA clock64 stamps written by the kernel itself
(drc_convg_set_timeline): setup (barrier initialisation) -> first operands landed -> last wgmma issued -> accumulator complete ->
last tile stored -> exit, averaged over the CTAs, plus the spread of CTA start times (globaltimer).  Not a timed number: the stamps
cost a few stores; the point is the breakdown."""
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from draco_b200.ops import conv as CV  # noqa: E402

dev = torch.device("cuda", 0)
lib = CV._lib()
lib.drc_convg_set_timeline.argtypes = [C.c_void_p]
lib.drc_convg_set_timeline.restype = None
MHZ = 1980.0                 # H100 SXM maximum SM clock (nvidia-smi clocks.max.sm); the stamps are clock64 cycles
SMS = torch.cuda.get_device_properties(dev).multi_processor_count   # the launch grid never exceeds one CTA per SM


def cl(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def wt(k, c, ks):
    return (torch.randn(k, c, ks, ks, device=dev) * 0.05).to(torch.bfloat16).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


rows = []
N = 128
for (c, k, hw, ks, st) in [(128, 128, 16, 3, 1), (256, 256, 8, 3, 1), (512, 512, 4, 3, 1), (128, 256, 16, 3, 2)]:
    x = cl(torch.randn(N, c, hw, hw, device=dev))
    w = wt(k, c, ks)
    dy = cl(torch.randn(N, k, hw // st, hw // st, device=dev))
    xbn = cl(torch.randn(N, c, hw, hw, device=dev))
    mean, invstd = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    for name, fn in (("fprop", lambda: CV.convg_tcgen05(x, w, (hw, hw), st)),
                     ("fprop+stats", lambda: CV.convg_tcgen05(x, w, (hw, hw), st, False, None, CV.BnStatRequest(1e-5, 0.1))),
                     ("dgrad", lambda: CV.convg_tcgen05(dy, w, (hw, hw), st, True)),
                     ("dgrad+bnbwd", (lambda: CV.convg_tcgen05(dy, w, (hw, hw), st, True, None, None, None,
                                                                (CV.BnBwdLink(xbn, mean, invstd, True), x))) if st == 1 else None)):
        if fn is None:
            continue
        for _ in range(3):
            fn()
        buf = torch.zeros(SMS * 8, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        lib.drc_convg_set_timeline(buf.data_ptr())
        fn()
        torch.cuda.synchronize()
        lib.drc_convg_set_timeline(None)
        t = buf.view(SMS, 8).cpu()
        t = t[t[:, 1] != 0]
        rel = (t[:, 1:7] - t[:, 1:2]).double() / MHZ           # us since CTA entry
        g0 = (t[:, 0] - t[:, 0].min()).double() / 1e3
        m = rel.mean(0)
        row = {"layer": [c, k, hw, ks, st], "op": name, "ctas": int(t.shape[0]), "cta_start_spread_us": round(float(g0.max()), 2),
               "setup_us": round(float(m[1]), 2), "first_operands_us": round(float(m[2]), 2),
               "last_mma_issued_us": round(float(m[3]), 2), "accumulator_ready_us": round(float(m[4]), 2),
               "tile_stored_us": round(float(m[5]), 2),
               "span_first_entry_to_last_exit_us": round(float((t[:, 7].max() - t[:, 0].min())) / 1e3, 2)}
        # the same launch five times back to back inside a CUDA graph: kernel period vs the time no CTA of either kernel is alive
        bufs = [torch.zeros(SMS * 8, dtype=torch.int64, device=dev) for _ in range(5)]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for b in bufs:
                lib.drc_convg_set_timeline(b.data_ptr())
                fn()
        lib.drc_convg_set_timeline(None)
        g.replay()
        torch.cuda.synchronize()
        tt = [b.view(SMS, 8).cpu() for b in bufs]
        tt = [x[x[:, 1] != 0] for x in tt]
        starts = [int(x[:, 0].min()) for x in tt]
        ends = [int(x[:, 7].max()) for x in tt]
        row["graph_period_us"] = round((starts[4] - starts[1]) / 3e3, 2)
        row["graph_dead_time_between_kernels_us"] = round(sum(starts[i + 1] - ends[i] for i in range(1, 4)) / 3e3, 2)
        rows.append(row)
        print(json.dumps(row), flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open("gpurun_out/conv_timeline.json", "w"), indent=1)
