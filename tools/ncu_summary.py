#!/usr/bin/env python3
"""Turns ncu output into small text summaries.

  ncu_summary.py launches <launches.csv>            per-kernel launch count, total/mean time and share of the GPU time
  ncu_summary.py report <file.ncu-rep>              key metrics of every kernel in a `--set full` report (needs ncu on PATH)
"""
import collections, csv, re, subprocess, sys

KEYS = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__occupancy_limit_registers",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
        "l1tex__t_sectors_pipe_lsu_mem_local_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_local_op_st.sum",
        "smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "sm__inst_executed.sum", "smsp__cycles_active.avg"]


def short(name):
    m = re.search(r"k_for_each<(?:arb::)?(\w+)>", name)
    return m.group(1) if m else re.sub(r"\(.*", "", name).replace("void ", "").replace("arb::", "")


def launches(path):
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    h = rows[0]; kn, mv, mn = h.index("Kernel Name"), h.index("Metric Value"), h.index("Metric Name")
    agg = collections.OrderedDict()
    for r in rows[1:]:
        if r[mn] != "gpu__time_duration.sum":
            continue
        a = agg.setdefault(short(r[kn]), [0, 0.0]); a[0] += 1; a[1] += float(r[mv].replace(",", "")) / 1e3
    total = sum(a[1] for a in agg.values())
    print("%-34s %8s %12s %12s %7s" % ("kernel", "launches", "total us", "mean us", "share"))
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("%-34s %8d %12.1f %12.1f %6.1f%%" % (k, n, us, us / n, 100 * us / total))
    print("%-34s %8d %12.1f" % ("TOTAL", sum(a[0] for a in agg.values()), total))


def report(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    h, units = rows[0], rows[1]
    for r in rows[2:]:
        print("== " + short(r[h.index("Kernel Name")]))
        for k in KEYS:
            if k in h:
                print("  %-82s %16s %s" % (k, r[h.index(k)], units[h.index(k)]))


if __name__ == "__main__":
    {"launches": launches, "report": report}[sys.argv[1]](sys.argv[2])
