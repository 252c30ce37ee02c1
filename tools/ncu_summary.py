"""Extract the headline metrics of every kernel in an .ncu-rep into a markdown table (run here, no GPU needed)."""
import csv
import io
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "time"),
    ("dram__bytes_read.sum", "dram rd"),
    ("dram__bytes_write.sum", "dram wr"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %"),
    ("lts__t_bytes.sum", "L2 bytes"),
    ("lts__t_sectors_srcunit_tex_op_read.sum", "L2->SM rd sectors (x32 B)"),
    ("lts__t_sector_hit_rate.pct", "L2 hit %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm %"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor %"),
    ("sm__inst_executed_pipe_tensor.sum", "tensor inst"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "occupancy %"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem"),
]


def main(rep, out, title):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    with open(out, "w") as fh:
        fh.write(f"# {title}\n\nsource: `{rep}` (`ncu --set full --clock-control none --import-source on`, one H100)\n\n")
        names = [lab for k, lab in KEYS if k in col]
        fh.write("| kernel | " + " | ".join(names) + " |\n|---|" + "---:|" * len(names) + "\n")
        for r in data:
            kn = r[col["Kernel Name"]].split("(")[0][-60:]
            vals = []
            for k, lab in KEYS:
                if k in col:
                    v, u = r[col[k]], units[col[k]]
                    try:
                        f = float(v.replace(",", ""))
                        if u in ("byte", "Kbyte", "Mbyte", "Gbyte"):
                            f *= {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
                            v = f"{f / 1e6:.2f} MB"
                        elif u in ("ns", "us", "usecond", "nsecond", "ms", "msecond"):
                            f *= {"ns": 1e-3, "nsecond": 1e-3, "us": 1, "usecond": 1, "ms": 1e3, "msecond": 1e3}[u]
                            v = f"{f:.2f} us"
                        elif u == "%":
                            v = f"{f:.1f}"
                        else:
                            v = f"{f:g}"
                    except ValueError:
                        pass
                    vals.append(v)
            fh.write(f"| `{kn}` | " + " | ".join(vals) + " |\n")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else sys.argv[1])
