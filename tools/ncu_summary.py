#!/usr/bin/env python
"""Summarise an .ncu-rep (read on the CPU box) into <name>.md: key raw metrics, the
top stall locations of the source page, and the occupancy / roofline lines of the details page.
    python tools/ncu_summary.py sgns_win.ncu-rep sgns_win_ncu.md "title" """
import csv
import io
import subprocess
import sys

WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
        "launch__block_size", "launch__shared_mem_per_block_dynamic", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__cycles_elapsed.avg.per_second",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sectors_srcunit_tex_op_red.sum", "lts__t_sectors.sum"]


def run(args):
    return subprocess.run(["ncu", "-i", *args], capture_output=True, text=True).stdout


def main():
    rep, out, title = sys.argv[1], sys.argv[2], (sys.argv[3] if len(sys.argv) > 3 else sys.argv[1])
    raw = list(csv.reader(io.StringIO(run([rep, "--page", "raw", "--csv"]))))
    lines = [f"# {title}", "", f"source: `{rep}` (ncu --set full --clock-control none --import-source on)", ""]
    if len(raw) >= 3:
        hdr, units = raw[0], raw[1]
        for row in raw[2:]:
            name = row[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
            lines += [f"## kernel `{name[:110]}`", "", "| metric | value | unit |", "|---|---|---|"]
            for h, u, v in zip(hdr, units, row):
                if h in WANT:
                    lines.append(f"| {h} | {v} | {u} |")
            lines.append("")
    det = run([rep, "--page", "details"])
    keep = [l.rstrip() for l in det.splitlines() if any(k in l for k in (
        "Duration", "DRAM Throughput", "L2 Hit Rate", "Registers Per Thread", "Theoretical Occupancy",
        "Achieved Occupancy", "Issued Warp Per Scheduler", "No Eligible", "Executed Ipc Active", "Memory Throughput",
        "L2 Cache Throughput", "Max Bandwidth", "Dynamic Shared Memory", "Block Size", "Grid Size", "Compute (SM) Throughput"))]
    lines += ["## details page (selected lines)", "", "```"] + keep[:40] + ["```", ""]
    src = list(csv.reader(io.StringIO(run([rep, "--page", "source", "--csv"]))))
    if len(src) > 2 and "# Samples" in src[1]:
        hdr = src[1]
        i_s, i_n = hdr.index("Source"), hdr.index("# Samples")
        stall_cols = [i for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
        rows = []
        for r in src[2:]:
            try:
                rows.append((int(r[i_n]), r))
            except (ValueError, IndexError):
                pass
        tot = sum(n for n, _ in rows) or 1
        lines += ["## top stall locations (SASS, warp-state samples)", "", "| % samples | instruction | dominant stall |", "|---|---|---|"]
        for n, r in sorted(rows, key=lambda x: -x[0])[:12]:
            dom = max(((int(r[i] or 0), hdr[i]) for i in stall_cols), default=(0, ""))
            lines.append(f"| {100 * n / tot:.1f} | `{r[i_s][:70]}` | {dom[1]} |")
        lines.append("")
    open(out, "w").write("\n".join(lines))
    print("written", out)


if __name__ == "__main__":
    main()
