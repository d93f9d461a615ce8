#!/usr/bin/env python
"""Per-kernel resource table from the ``-Xptxas -v`` output of the in-tree build (``build/obj/*.log``, written by
``distributedmnist_b200/ops/build.py``): registers, static shared memory, stack / spill bytes, barriers.  No GPU needed.

    python tools/ptxas_report.py [out.txt]

Why it is tracked: co-residency of the step's kernels is a register / shared-memory budget (4 x 16 K registers per SM
sub-partition, one shared-memory carve-out for all of them), and a spill in a wgmma accumulator is a silent 2x.
"""
from __future__ import annotations

import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def demangle(names):
    try:
        out = subprocess.run(["c++filt"] + names, capture_output=True, text=True, check=True).stdout.splitlines()
        return [re.sub(r"\(.*$", "", o.replace("void ", "")) for o in out]
    except Exception:
        return names


def parse(path):
    rows, cur = [], None
    for line in open(path):
        m = re.search(r"Compiling entry function '(\S+)' for '(\S+)'", line)
        if m:
            cur = {"name": m.group(1), "arch": m.group(2), "stack": 0, "spill_st": 0, "spill_ld": 0, "regs": 0, "barriers": 0,
                   "smem": 0}
            rows.append(cur)
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            cur["stack"], cur["spill_st"], cur["spill_ld"] = map(int, m.groups())
        m = re.search(r"Used (\d+) registers", line)
        if m:
            cur["regs"] = int(m.group(1))
            b = re.search(r"used (\d+) barriers", line)
            cur["barriers"] = int(b.group(1)) if b else 0
            s = re.search(r"(\d+) bytes smem", line)
            cur["smem"] = int(s.group(1)) if s else 0
    return rows


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    lines = ["# -Xptxas -v of the shipped library (sm_90a); dynamic shared memory is set at launch and not listed here",
             "%-14s %-78s %5s %7s %6s %9s %4s" % ("file", "kernel", "regs", "smem_B", "stack", "spill_B", "bar")]
    spills = 0
    for log in sorted(glob.glob(os.path.join(ROOT, "build", "obj", "*.log"))):
        rows = parse(log)
        names = demangle([r["name"] for r in rows]) if rows else []
        for r, nm in zip(rows, names):
            sp = r["spill_st"] + r["spill_ld"]
            spills += sp
            lines.append("%-14s %-78s %5d %7d %6d %9d %4d" % (os.path.basename(log)[:-4], nm[:78], r["regs"], r["smem"], r["stack"],
                                                            sp, r["barriers"]))
    lines.append("# total spill bytes over all kernels: %d" % spills)
    text = "\n".join(lines) + "\n"
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(text)
    sys.stdout.write(text)


if __name__ == "__main__":
    main()
