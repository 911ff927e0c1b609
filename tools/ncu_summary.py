"""ncu report -> markdown table of the metrics the roofline discussion uses.
  ncu -i cg.ncu-rep --page raw --csv > raw.csv ; python tools/ncu_summary.py raw.csv names.txt > ncu_cg.md"""
import csv, sys

WANT = [("gpu__time_duration.sum", "us", 1.0),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor %", 1.0),
        ("l1tex__m_xbar2l1tex_read_bytes.sum", "L2->SM MB", 1.0),
        ("dram__bytes_read.sum", "dram rd MB", 1.0), ("dram__bytes_write.sum", "dram wr MB", 1.0),
        ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 %", 1.0),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %", 1.0),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps %", 1.0),
        ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "long_sb / issue", 1.0),
        ("launch__grid_size", "grid", 1.0), ("launch__registers_per_thread", "regs", 1.0)]
rows = list(csv.reader(open(sys.argv[1])))
hdr, units = rows[0], rows[1]
names = [l.strip() for l in open(sys.argv[2])] if len(sys.argv) > 2 else None
cols = [(hdr.index(m), lab, units[hdr.index(m)]) for m, lab, _ in WANT if m in hdr]
print("| launch | " + " | ".join(lab for _, lab, _ in cols) + " |")
print("|---|" + "---|" * len(cols))
for i, r in enumerate(rows[2:]):
    vals = []
    for ci, lab, unit in cols:
        v = r[ci].replace(",", "")
        try:
            f = float(v)
            if lab == "us" and unit == "ns":
                f /= 1e3
            if "MB" in lab and unit == "byte":
                f /= 1e6
            if "MB" in lab and unit == "Kbyte":
                f /= 1e3
            v = f"{f:.1f}" if abs(f) < 1e5 else f"{f:.0f}"
        except ValueError:
            pass
        vals.append(v)
    print(f"| {names[i] if names and i < len(names) else i} | " + " | ".join(vals) + " |")
