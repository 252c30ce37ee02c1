"""Per-kernel table of the Hopper-specific SASS opcodes in the built library (cuobjdump -sass): wgmma (HGMMA), wgmma fences /
waits (WARPGROUP.*), TMA loads / stores (UTMALDG / UTMASTG, .MULTICAST), mbarrier ops (SYNCS.*), cluster barriers (UCGABAR_*),
bulk copies, multimem and system-scope accesses.  Prints a markdown table.

    python tools/sass_ops.py [path/to/libdraco_cuda.so] > kernel_hopper_ops.md
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "draco_b200", "_lib", "libdraco_cuda.so")
KEEP = re.compile(r"^(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UTMAPF|SYNCS|UCGABAR|UBLKCP|MULTIMEM|CCTL\.IVALL|"
                  r"(LDG|STG|ATOMG|RED|LD|ST|ATOM)\.[A-Z0-9.]*(SYS|STRONG\.GPU)|MEMBAR|ERRBAR|ACQBULK|ARRIVES|UTMACMDFLUSH|UTMACCTL)")
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
filt = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True, text=True).stdout.split("\n")
names = dict(zip(re.findall(r"Function : (\S+)", sass), filt))
per = collections.OrderedDict()
cur = None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        n = names.get(m.group(1), m.group(1))
        n = re.sub(r"\(anonymous namespace\)::", "", n)
        n = re.sub(r"\(.*$", "", n).replace("void ", "")
        cur = per.setdefault(n, collections.Counter())
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
    if m and cur is not None and KEEP.match(m.group(1)):
        cur[m.group(1)] += 1
out = ["# Hopper-specific SASS opcodes per kernel of `libdraco_cuda.so` (cuobjdump -sass, sm_90a; `tools/sass_ops.py`)", "",
       "`HGMMA` = wgmma.mma_async, `WARPGROUP.*` = wgmma fence / commit / wait, `UTMALDG` / `UTMASTG` = TMA tensor load / store",
       "(`.MULTICAST`), `SYNCS.*` = mbarrier ops, `UCGABAR_*` = cluster barrier, `UBLKCP` = cp.async.bulk, `*.SYS` = system-scope",
       "accesses (peer memory flags / stores), `MULTIMEM` = NVLS multicast stores.", "",
       "| kernel | opcodes (count) |", "|---|---|"]
for n in sorted(per):
    if per[n]:
        out.append(f"| `{n}` | " + ", ".join(f"`{k}` x{v}" for k, v in sorted(per[n].items())) + " |")
print("\n".join(out))
print(f"{sum(1 for n in per if per[n])} kernels with Hopper-specific opcodes of {len(per)}", file=sys.stderr)
