"""Summarise a `bench.py --timeline` kernel timeline (one rank): step period, busy time per stream, time per kernel class, and
the forward / backward / tail split of the middle one of the three recorded steps.

    python tools/summarize_timeline.py timeline.rank1.txt > step_timeline_worker.md
"""
import collections
import re
import sys

rows = []
for line in open(sys.argv[1]).read().splitlines()[1:]:
    p = line.split(None, 4)
    rows.append((float(p[0]), float(p[1]), p[3], p[4]))
starts = [i for i, r in enumerate(rows) if r[3].startswith("wait_flags_kernel")]
if len(starts) < 3:
    starts = [0, len(rows) // 3, 2 * len(rows) // 3]
# the recorded step with the shortest period (a profiler flush can stall one of the three for milliseconds)
cands = [(rows[starts[i + 1]][0] - rows[starts[i]][0], starts[i], starts[i + 1]) for i in range(len(starts) - 1)]
_, a, b = min(cands) if cands else (0, starts[1], len(rows))
step = rows[a:b]
t0 = step[0][0]
period = rows[b][0] - t0 if b < len(rows) else step[-1][0] + step[-1][1] - t0


def cls(n):
    n = n.replace("(anonymous namespace)::", "").replace("void ", "")
    for pat, c in (("conv_halo_wgmma_kernel<false>|conv_halo_wgmma_kernel<0>", "conv fprop (halo, wgmma)"),
                   ("conv_halo_wgmma_kernel", "conv dgrad (halo, wgmma)"),
                   ("wgrad_halo|convg_wgrad|wgradg_reduce|stem_wgrad", "conv wgrad (wgmma / stem) + split-K fold"),
                   (r"convg_wgmma_kernel<\d+, \d+, false|convg_wgmma_kernel<\d+, \d+, 0", "conv fprop (tap, wgmma)"),
                   ("convg_wgmma_kernel", "conv dgrad (tap, wgmma)"),
                   ("stem_fprop", "stem fprop"),
                   ("bn_apply", "BatchNorm apply (+res +ReLU)"), ("bn_bwd", "BatchNorm backward"), ("bn_stats", "BatchNorm statistics"),
                   ("gemm_bf16", "linear (wgmma GEMM)"), ("push_encode", "push_encode (gradient -> PS slot)"),
                   ("ce_fused|prep_input|gap_|head_prep|cast_params|wait_flags|stamp|step_add|dropout", "loss / prep / pool / flags (ours)"),
                   ("Memcpy|memset|Memset", "memcpy / memset")):
        if re.search(pat, n):
            return c
    return "ATen elementwise / reduce"


by = collections.OrderedDict()
for r in step:
    c = cls(r[3])
    d = by.setdefault(c, [0.0, 0])
    d[0] += r[1]
    d[1] += 1
busy = collections.Counter()
for r in step:
    busy[r[2]] += r[1]
first_bwd = next((r[0] for r in step if "bn_bwd" in r[3] or "gap_bwd" in r[3]), None)
last_main = max(r[0] + r[1] for r in step if "push_encode" not in r[3])
print(f"# Kernel timeline of one training step ({sys.argv[1].split('/')[-1]}, CUPTI through torch.profiler, CUDA-graph replay)\n")
print(f"step period {period:.0f} us; {len(step)} kernels; busy time per stream: "
      + ", ".join(f"stream {k}: {v:.0f} us" for k, v in busy.most_common()) + "\n")
if first_bwd is not None:
    print(f"forward 0 -> {first_bwd - t0:.0f} us, backward -> {last_main - t0:.0f} us, tail (last push, flags, next-step staging) -> {period:.0f} us\n")
print("| kernel class | total us | launches |\n|---|---:|---:|")
for c, (t, n) in sorted(by.items(), key=lambda kv: -kv[1][0]):
    print(f"| {c} | {t:.0f} | {n} |")
print(f"| **sum of kernel durations** | {sum(v[0] for v in by.values()):.0f} | {len(step)} |")
