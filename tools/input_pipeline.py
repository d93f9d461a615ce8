#!/usr/bin/env python
"""Does the trainer keep up with the engine?  Host-fed batches versus ``--device_data`` through ``train.train()`` itself, on
one GPU.  Prints one JSON line.

Each run trains LeNet with B = 256, K = N = 1 on a synthetic 60 000-row set for ``--steps`` steps (``--log_every=1000``, no
checkpoint inside the run).  The two input paths alternate for ``--rounds`` rounds in one invocation, so the spread
between rounds shows next to the difference between the paths.  Per run:

* trainer images/s: the host clock at the log line of iteration ``--window-from`` and at the last log line (each written
  right after the host waited for that step's completion event), over the images trained in between;
* host CPU seconds per step: ``time.process_time()`` at the same two points (all threads of the process: the batch
  packer's helper threads included), over the steps in between.

``bench.py --gpus 1`` runs once for the engine's device rate (graph replays of pre-packed batches) and its end-to-end rate.

    python tools/input_pipeline.py [--steps 10000] [--rounds 3] [--trace DIR] [--out results/input_pipeline.json]

``--trace DIR``: after the timed runs, a ``torch.profiler`` timeline (CUDA activities) of a short run of each path, written
to ``DIR/trace_host.json`` / ``DIR/trace_device_data.json``, with the gather kernel's duration and the idle gap between
one step's last kernel and the next step's first kernel (median and 90th percentile over the run's last steps).
"""
import argparse
import json
import logging
import os
import re
import subprocess
import sys
import tempfile
import time

import gpu_timing
import numpy as np
import torch
from distributedmnist_b200.data import DataSet, make_synthetic_mnist
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import train

B = 256
_STEP_LINE = re.compile(r"Worker 0: .*: step ([0-9]+), loss = ")


class _Stamps(logging.Handler):
    """(step, host clock, process CPU time) at every per-step log line of the chief."""

    def __init__(self):
        super().__init__()
        self.rows = []

    def emit(self, record):
        m = _STEP_LINE.match(record.getMessage())
        if m:
            self.rows.append((int(m.group(1)), time.perf_counter(), time.process_time()))


def run(ctx, table, device_data: bool, steps: int, window_from: int):
    x, y = table
    FLAGS.reset()
    with tempfile.TemporaryDirectory() as d:
        FLAGS.parse(["--train_dir=%s" % d, "--batch_size=%d" % B, "--max_steps=%d" % steps, "--model=lenet",
                     "--log_every=1000", "--save_interval_secs=1e9", "--save_results_period=1000000000",
                     "--device_data=%s" % ("true" if device_data else "false")])
        ds = DataSet(x, y, seed=4321)
        stamps = _Stamps()
        log = logging.getLogger("dmnist")
        log.addHandler(stamps)
        try:
            res = train(ctx, ds, None, FLAGS)
        finally:
            log.removeHandler(stamps)
        del res
    torch.cuda.synchronize()
    rows = [r for r in stamps.rows if r[0] >= window_from]
    (s0, t0, c0), (s1, t1, c1) = rows[0], rows[-1]
    return {"images_per_s": B * (s1 - s0) / (t1 - t0), "cpu_s_per_step": (c1 - c0) / (s1 - s0), "window_steps": s1 - s0,
            "window_s": t1 - t0}


def bench_rate(steps: int):
    r = subprocess.run([sys.executable, os.path.join(gpu_timing.ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps),
                        "--warmup", "200"], capture_output=True, text=True, cwd=tempfile.gettempdir())
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not line:
        raise RuntimeError("bench.py failed:\n" + (r.stdout + r.stderr)[-3000:])
    out = json.loads(line[-1])
    return {"device_images_per_s": out["value"], "device_ms_per_step": out["ms_per_step"],
            "e2e_images_per_s": out["e2e"]["value"], "e2e_ms_per_step": out["e2e"]["ms_per_step"]}


def _pct(v, q):
    return float(np.percentile(np.asarray(v, np.float64), q)) if v else None


def trace(ctx, table, device_data: bool, path: str, steps: int = 400, last: int = 200):
    """Timeline of a short run; kernel statistics of its last `last` steps."""
    from torch.profiler import ProfilerActivity, profile
    x, y = table
    FLAGS.reset()
    with tempfile.TemporaryDirectory() as d:
        FLAGS.parse(["--train_dir=%s" % d, "--batch_size=%d" % B, "--max_steps=%d" % steps, "--model=lenet",
                     "--log_every=1000", "--save_interval_secs=1e9", "--save_results_period=1000000000",
                     "--device_data=%s" % ("true" if device_data else "false")])
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            train(ctx, DataSet(x, y, seed=4321), None, FLAGS)
            torch.cuda.synchronize()
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy")]
    ev.sort(key=lambda e: e["ts"])
    kern = [e for e in ev if e["cat"] == "kernel"]
    gather = [e for e in kern if "gather_batch" in e["name"]]
    step_kern = [e for e in kern if "gather_batch" not in e["name"]]
    starts = [i for i, e in enumerate(step_kern) if "conv1_fwd" in e["name"]][-(last + 1):]
    gaps, periods = [], []
    for a, b in zip(starts, starts[1:]):
        end_prev = max(e["ts"] + e["dur"] for e in step_kern[a:b])       # the previous step's last kernel to finish
        gaps.append(step_kern[b]["ts"] - end_prev)
        periods.append(step_kern[b]["ts"] - step_kern[a]["ts"])
    h2d = [e["dur"] for e in ev if e["cat"] == "gpu_memcpy" and "HtoD" in e["name"]][-last:]
    g = [e["dur"] for e in gather][-last:]
    return {"trace": path, "steps_measured": len(gaps),
            "step_period_us_median": _pct(periods, 50), "gap_us_median": _pct(gaps, 50), "gap_us_p90": _pct(gaps, 90),
            "gather_us_median": _pct(g, 50), "gather_us_p90": _pct(g, 90),
            "h2d_copy_us_median": _pct(h2d, 50)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10000)
    ap.add_argument("--window-from", type=int, default=1000, help="first logged step of the timed window")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bench-steps", type=int, default=3000)
    ap.add_argument("--trace", default="", metavar="DIR")
    ap.add_argument("--out", default=os.path.join("results", "input_pipeline.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        sys.exit(1)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    info = gpu_timing.card()
    ctx = init_context(FLAGS)
    tr_x, tr_y, _, _ = make_synthetic_mnist(60000, 10, seed=1234)
    table = (tr_x, tr_y)
    runs = {"host": [], "device_data": []}
    for _ in range(args.rounds):
        for name in ("host", "device_data"):
            runs[name].append(run(ctx, table, name == "device_data", args.steps, args.window_from))
    out = dict(info, batch=B, steps=args.steps, window_from=args.window_from, rounds=args.rounds, runs=runs)
    for name, rs in runs.items():
        ips = [r["images_per_s"] for r in rs]
        cpu = [r["cpu_s_per_step"] * 1e6 for r in rs]
        out[name] = {"images_per_s_median": float(np.median(ips)), "images_per_s_min": min(ips), "images_per_s_max": max(ips),
                     "cpu_us_per_step_median": float(np.median(cpu)), "cpu_us_per_step_min": min(cpu),
                     "cpu_us_per_step_max": max(cpu)}
    out["bench"] = bench_rate(args.bench_steps)
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
        out["trace"] = {name: trace(ctx, table, name == "device_data", os.path.join(args.trace, "trace_%s.json" % name))
                        for name in ("host", "device_data")}
    gpu_timing.emit(out, args.out)


if __name__ == "__main__":
    main()
