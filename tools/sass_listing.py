#!/usr/bin/env python
"""Committed SASS evidence: full instruction listings of the hot kernels of ``libdmnist_b200.so`` (``cuobjdump -sass``, hex
encodings stripped) plus a per-kernel count of the mnemonics that prove a Hopper-native kernel
(``HGMMA`` = wgmma.mma_async, ``WARPGROUP`` = wgmma fence / wait, ``WARPGROUP.DEPBAR.LE gsb0, 0x0`` = wait for every
wgmma in flight (one per HGMMA means ptxas serialized the kernel), ``LDSM`` = ldmatrix, ``UTMALDG``/``UBLKCP`` = TMA, ``LDGMC`` =
multimem.ld_reduce (a ``multimem.st`` is an ordinary ``STG.E.128.STRONG.SYS`` whose ADDRESS is the multicast mapping),
``SYNCS`` = mbarrier).  Needs no GPU:  ``python tools/sass_listing.py [DEST]`` (default results/sass)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "distributedmnist_b200", "lib", "libdmnist_b200.so")
HOT = [("conv2_fwd", r"conv2_fwd_kernel"), ("conv2_dgrad", r"conv2_dgrad_kernel"), ("conv2_wgrad", r"conv2_wgrad_kernel"),
       ("conv1_fwd_tc", r"conv1_fwd_tc_kernel"), ("conv1_wgrad_tc", r"conv1_wgrad_tc_kernel"),
       ("gemm_fc1_fwd", r"gemm_tc_kernelILi64ELb0ELb1ELi0E"), ("gemm_fc1_dgrad_unpool", r"gemm_tc_kernelILi64ELb0ELb0ELi4E"),
       ("gemm_fc1_wgrad_bf16", r"gemm_tc_kernelILi128ELb1ELb1ELi2E"), ("bucket_early_n8", r"bucket_early_kernelILi8E"),
       ("bucket_late_ll", r"bucket_late_ll_kernel"), ("fused_sync_sgd_kofn", r"fused_sync_sgd_kernelILb1E"),
       ("iv_apply", r"iv_apply_kernel")]
KEY = [("wgmma", r"\bHGMMA"), ("wgmma fence/wait", r"\bWARPGROUP"), ("wgmma wait-all", r"\bWARPGROUP\.DEPBAR\.LE gsb0, 0x0\b"),
       ("ldmatrix", r"\bLDSM"),
       ("TMA tensor load", r"\bUTMALDG"), ("TMA bulk", r"\bUBLKCP"), ("mbarrier", r"\bSYNCS"), ("multimem ld_reduce", r"\bLDGMC|\bLD\S*\.MC|MULTIMEM|REDUX\.MC"),
       ("st.sys (incl. multimem.st)", r"\bSTG?\.E\S*\.STRONG\.SYS"), ("legacy HMMA (must be 0)", r"\bHMMA"), ("fence.sys", r"MEMBAR\S*\.SYS|FENCE\S*SYS"),
       ("sys-scope ld/st", r"\b(LD|ST)G?\S*\.SYS")]


def main():
    dest = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "results", "sass")
    os.makedirs(dest, exist_ok=True)
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    funcs = {}
    cur = None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);\s*/\*", line)
        if m:
            funcs[cur].append("/*%s*/ %s" % (m.group(1), m.group(2).strip()))
    summary = ["# SASS summary of %s (cuobjdump -sass; counts of the Hopper-specific mnemonics per kernel)" % os.path.relpath(LIB, ROOT),
               "%-26s %7s " % ("kernel", "instrs") + " ".join("%18s" % k for k, _ in KEY)]
    for short, pat in HOT:
        names = [f for f in funcs if re.search(pat, f)]
        if not names:
            summary.append("%-26s (not found: %s)" % (short, pat))
            continue
        body = funcs[names[0]]
        with open(os.path.join(dest, short + ".sass"), "w") as f:
            f.write("// %s\n// %d instructions; cuobjdump -sass %s (encodings stripped)\n" % (names[0], len(body), os.path.relpath(LIB, ROOT)))
            f.write("\n".join(body) + "\n")
        counts = [sum(1 for ins in body if re.search(rx, ins)) for _, rx in KEY]
        summary.append("%-26s %7d " % (short, len(body)) + " ".join("%18d" % c for c in counts))
    with open(os.path.join(dest, "SUMMARY.txt"), "w") as f:
        f.write("\n".join(summary) + "\n")
    print("\n".join(summary))


if __name__ == "__main__":
    main()
