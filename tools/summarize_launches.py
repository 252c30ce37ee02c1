"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch log into a markdown table."""
import collections
import csv
import re
import sys


def main(path, out, title):
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    agg, tot, n = collections.OrderedDict(), 0.0, 0
    for row in csv.DictReader(lines):
        if row.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(row["Metric Value"].replace(",", ""))
        v = v / 1e3 if row["Metric Unit"] == "ns" else v * 1e3 if row["Metric Unit"] == "ms" else v
        name = re.sub(r"^void ", "", row["Kernel Name"]).replace("<unnamed>::", "").replace("(anonymous namespace)::", "")
        name = re.sub(r"\(.*$", "", name)                       # drop the argument list, keep template arguments
        name = re.sub(r"^at::native::(\(anonymous namespace\)::)?", "at::", name)
        name = re.sub(r"<.*", "", name)[:90] if name.startswith("at::") else name[:90]
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1; a[1] += v; tot += v; n += 1
    with open(out, "w") as fh:
        fh.write(f"# {title}\n\nsource: `{path}` (ncu, serialised, cold caches: compare shares, not absolutes)\n\n")
        fh.write(f"total: {n} launches, {tot / 1e3:.2f} ms\n\n| share | total us | launches | kernel |\n|---:|---:|---:|---|\n")
        for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:45]:
            fh.write(f"| {100 * t / tot:.1f}% | {t:.1f} | {c} | `{k}` |\n")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else "kernel launches")
