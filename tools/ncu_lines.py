#!/usr/bin/env python3
"""Per-source-line view of one kernel of an `ncu --set full` report: the SASS rows of `ncu --page source` are joined (by instruction index) with the line
table of the same kernel in the cubin (`nvdisasm -g`), and instructions / thread instructions / stall samples are summed per source line.

  ncu_lines.py <report.ncu-rep> <kernel name regex> <file.cubin> [top N]
The cubin must come from the build that was profiled (cuobjdump -xelf all libarriba_b200.so)."""
import csv, os, re, subprocess, sys, collections

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "arriba_b200", "csrc")


def main():
    rep, kern, cubin = sys.argv[1:4]
    top = int(sys.argv[4]) if len(sys.argv) > 4 else 40
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--kernel-name", "regex:" + kern], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr = next(i for i, r in enumerate(rows) if "Instructions Executed" in r)
    h = rows[hdr]
    ie, te, sm, src = h.index("Instructions Executed"), h.index("Thread Instructions Executed"), h.index("# Samples"), h.index("Source")
    inst = []
    for r in rows[hdr + 1:]:
        if len(r) <= te or not r[0].startswith("0x"):
            if inst and len(r) > 1 and r[0] == "Kernel Name":
                break   # next kernel instance
            continue
        inst.append((int(r[ie]), int(r[te]), int(r[sm]), r[src].strip()))
    dis = subprocess.run(["nvdisasm", "-g", "-c", cubin], stdout=subprocess.PIPE, text=True).stdout
    # find the function section whose name matches
    lines = dis.splitlines()
    start = next(i for i, l in enumerate(lines) if l.startswith(".text.") and re.search(kern, l))
    cur = ("?", 0); table = []
    for l in lines[start + 1:]:
        if l.startswith(".text.") or l.startswith(".section"):
            if table:
                break
        m = re.search(r'//## File "([^"]+)", line (\d+)', l)
        if m:
            cur = (m.group(1).split("/")[-1], int(m.group(2)))
            # inlined-at chain: keep the innermost (first) location
            continue
        if re.match(r"\s+/\*[0-9a-f]{4}\*/", l):
            table.append(cur)
    n = min(len(inst), len(table))
    if len(inst) != len(table):
        print("warning: %d profiled instructions vs %d in the cubin" % (len(inst), len(table)))
    agg = collections.OrderedDict()
    for k in range(n):
        a = agg.setdefault(table[k], [0, 0, 0]); a[0] += inst[k][0]; a[1] += inst[k][1]; a[2] += inst[k][2]
    ti, tt, ts = sum(a[0] for a in agg.values()), sum(a[1] for a in agg.values()), sum(a[2] for a in agg.values())
    print("warp instructions %d, thread instructions %d (%.1f lanes), samples %d" % (ti, tt, tt / max(1, ti), ts))
    srcs = {}
    for (f, ln), a in sorted(agg.items(), key=lambda kv: -kv[1][2])[:top]:
        if f not in srcs:
            try:
                srcs[f] = open(next(p for p in (os.path.join(CSRC, f), os.path.join(CSRC, "host", f)) if os.path.exists(p))).read().splitlines()
            except Exception:
                srcs[f] = []
        text = srcs[f][ln - 1].strip()[:110] if 0 < ln <= len(srcs[f]) else ""
        print("%5.1f%% smp %5.1f%% inst %4.1f lanes  %s:%d  %s" % (100.0 * a[2] / max(1, ts), 100.0 * a[0] / max(1, ti), a[1] / max(1, a[0]), f, ln, text))


if __name__ == "__main__":
    main()
