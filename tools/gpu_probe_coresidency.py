"""Do CTAs of different kernels share an SM?  Launch a resident kernel (1 CTA/SM, spinning 60 us) and a guest kernel on
another stream; report when the guest's CTAs started relative to the residents (csrc/probes/coresidency_probe.cu)."""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from distributedmnist_b200.ops.lib import check, load, ptr  # noqa: E402

from distributedmnist_b200.ops.build import build_probes  # noqa: E402

lib = ctypes.CDLL(build_probes())       # the probes live in their own library (csrc/probes/)
n = torch.cuda.get_device_properties(0).multi_processor_count   # one resident CTA per SM
out = torch.zeros(5, dtype=torch.int64, device="cuda")
sink = torch.zeros(4, device="cuda")
lo, hi = 0, -1
rows = []
cases = [
    # name, res_smem, res_regs, res_ctas, guest_thr, guest_ctas, pdl, prio_res, prio_guest, carve_res, carve_guest
    ("small resident (0 KB, 16 regs)", 0, 16, n, 128, n, 0, lo, lo, -1, -1),
    ("100 KB smem", 100 << 10, 16, n, 128, n, 0, lo, lo, -1, -1),
    ("196 KB smem", 196 << 10, 16, n, 128, n, 0, lo, lo, -1, -1),
    ("196 KB smem, both carve-out 100", 196 << 10, 16, n, 128, n, 0, lo, lo, 100, 100),
    ("196 KB smem, 200+ regs", 196 << 10, 200, n, 128, n, 0, lo, lo, -1, -1),
    ("196 KB, 200+ regs, resident high prio / guest low", 196 << 10, 200, n, 128, n, 0, hi, lo, -1, -1),
    ("196 KB, 200+ regs, PDL attribute on both", 196 << 10, 200, n, 128, n, 1, hi, lo, -1, -1),
    ("196 KB, 200+ regs, guest 256 thr x 64 CTAs", 196 << 10, 200, n, 256, 64, 0, hi, lo, -1, -1),
    ("0 KB, 200+ regs", 0, 200, n, 128, n, 0, lo, lo, -1, -1),
    ("196 KB, 90 regs", 196 << 10, 100, n, 128, n, 0, lo, lo, -1, -1),
    ("all SMs but 4 resident (196 KB, 200 regs)", 196 << 10, 200, n - 4, 128, n, 0, hi, lo, -1, -1),
]
for c in cases:
    name, args = c[0], c[1:]
    for rep in range(2):
        check(lib.dm_probe_coresidency(*args, 0, ptr(out), ptr(sink)), "probe")
    t = out.cpu().tolist()
    r0 = t[0]
    rows.append("%-58s resident %5.1f us | guest first start +%5.1f us, last start +%5.1f us, last end +%5.1f us  -> %s"
                % (name, (t[1] - r0) / 1e3, (t[2] - r0) / 1e3, (t[3] - r0) / 1e3, (t[4] - r0) / 1e3,
                   "CO-RESIDENT" if t[3] < t[1] - 5000 else ("partly" if t[2] < t[1] - 5000 else "only after the residents exit")))
    print(rows[-1], flush=True)
os.makedirs("results", exist_ok=True)
open("results/coresidency_probe.txt", "w").write("\n".join(rows) + "\n")
