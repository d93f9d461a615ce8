#!/usr/bin/env python
"""Experiment driver + plots: run a list of configurations for N global steps each, scrape the logs,
draw time-to-accuracy / step-rate / loss curves and the straggler compute-time CDF.

reference: tools/benchmark.py --
``load_cfg_from_file`` (:13-15), ``run_tf_and_download_files`` with the ``step N,`` regex poll
(:24-58), the evaluator/ELAPSED TIMES scrapers (:60-163), the five figures ``time_loss.png``,
``time_step.png``, ``time_precision.png``, ``step_losses.png``, ``time_cdfs.png`` and the percentile
report (:60-111, 165-263), ``plot_figs`` (:265-279) and the ``use_dir`` / ``select_files`` CLI (:281-292).
Differences: the fleet is one box (tools/cluster.py), polling is every second instead of every 60 s
(a 300-step run takes seconds on H100, not minutes), figures are written by a dependency-free
rasteriser when matplotlib is absent, and the time-CDF plot is enabled.
"""
from __future__ import annotations

import ast
import glob
import json
import os
import re
import sys
import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cluster import Cfg, cluster_run  # noqa: E402
from distributedmnist_b200.utils.miniplot import line_plot  # noqa: E402


def load_cfg_from_file(cfg_file: str) -> Cfg:
    """Configuration files are Python literals ``Cfg({...})`` (reference: ``eval`` of the file)."""
    with open(cfg_file) as f:
        src = f.read()
    tree = ast.parse(src.strip(), mode="eval")
    call = tree.body
    if not (isinstance(call, ast.Call) and getattr(call.func, "id", "") == "Cfg" and len(call.args) == 1):
        raise ValueError("%s: expected a single Cfg({...}) literal" % cfg_file)
    from cluster import cfg as default_cfg
    merged = dict(default_cfg)          # raw (un-interpolated) defaults, then the file's overrides
    merged.update(ast.literal_eval(call.args[0]))
    if os.environ.get("DMNIST_CLAMP_GPUS", "0") == "1" and merged.get("n_gpus"):
        # dry runs of an 8-GPU matrix on a smaller box: as many replicas as there are GPUs, K clamped accordingly
        from cluster import n_gpus_available
        have = n_gpus_available()
        if have and merged["n_masters"] + merged["n_workers"] > have:
            merged["n_workers"] = max(have - merged["n_masters"], 0)
            k = int(merged.get("num_replicas_to_aggregate", have))
            merged["num_replicas_to_aggregate"] = str(min(k, have))
    return Cfg(merged)


def current_iteration(path: str) -> int:
    cur = 0
    try:
        with open(path) as f:
            for line in f:
                m = re.match(r".*step ([0-9]*),.*", line)
                if m and m.group(1):
                    cur = max(cur, int(m.group(1)))
    except OSError:
        pass
    return cur


def shutdown_and_launch(cfg: Cfg) -> None:
    """reference tools/benchmark.py:17-22: tear the fleet down and bring a fresh one up.  On one box that is: stop every
    role of the configuration, then ``launch`` (creates the run directory -- the stand-in for the NFS mount)."""
    cluster_run(["cluster.py", "shutdown"], cfg)
    cluster_run(["cluster.py", "launch"], cfg)


def check_if_reached_iters(cluster_string: str, n_iters: int, cfg: Cfg, master_file_name: str = "out_master",
                           outdir: str = "/tmp/") -> bool:
    """reference :24-34: fetch the master's log and report whether it has passed ``n_iters`` global steps."""
    fname = cluster_run(["cluster.py", "download_file", cluster_string, master_file_name, outdir], cfg)
    cur = current_iteration(fname)
    print("Currently on iteration %d" % cur)
    return cur > n_iters


def run_tf_and_download_files(n_iters: int, cfg: Cfg, evaluator_file_name: str = "out_evaluator",
                              master_file_name: str = "out_master", outdir: str = "result_dir",
                              timeout_s: float = 3600.0, poll_s: float = 1.0) -> Dict:
    cluster_run(["cluster.py", "kill_all_python"], cfg)
    spec = cluster_run(["cluster.py", "run_tf"], cfg)
    master = os.path.join(cfg["base_out_dir"], master_file_name)
    t0 = time.time()
    while current_iteration(master) <= n_iters:
        if time.time() - t0 > timeout_s:
            print("timeout waiting for %s to reach step %d" % (cfg["name"], n_iters))
            break
        live = cluster_run(["cluster.py", "list_running_instances"], cfg)
        if "master" not in live:
            break                      # run finished on its own (max_steps reached)
        time.sleep(poll_s)
    print("Currently on iteration %d" % current_iteration(master))
    time.sleep(2 * poll_s)             # let the evaluator pick up the last checkpoint
    cluster_run(["cluster.py", "kill_all_python"], cfg)
    for fname in (evaluator_file_name, master_file_name):
        try:
            cluster_run(["cluster.py", "download_file", spec["cluster_string"], fname, outdir], cfg)
        except OSError as e:
            print("could not download %s: %s" % (fname, e))
    return spec


# ---- scrapers ---------------------------------------------------------------------------------------
def extract_times_losses_precision(fname: str) -> Tuple[List[float], List[float], List[float], List[int]]:
    times, losses, precisions, steps = [], [], [], []
    with open(fname) as f:
        for line in f:
            m = re.match(r"Num examples: ([0-9]*)  Precision @ 1: ([\.0-9]*) Loss: ([\.0-9]*) Time: ([\.0-9]*)", line)
            sm = re.match(r".* step=([0-9]*)", line)
            if m:
                precisions.append(float(m.group(2)))
                losses.append(float(m.group(3)))
                times.append(float(m.group(4)))
            if sm:
                steps.append(int(sm.group(1)))
    n = min(len(times), len(losses), len(precisions), len(steps))
    return times[:n], losses[:n], precisions[:n], steps[:n]


def extract_compute_times(fname: str) -> List[Tuple[float, int, int]]:
    """Last ``ELAPSED TIMES [(secs, worker, iteration), ...]`` line of a master log."""
    out: List[Tuple[float, int, int]] = []
    with open(fname) as f:
        for line in f:
            m = re.match(r".*ELAPSED TIMES (.*)", line)
            if m:
                out = ast.literal_eval(m.group(1))
    return out


def extract_compute_times_no_master(fname: str, exclude_workers: Sequence[int] = (0,)) -> List[Tuple[float, int, int]]:
    """reference :124-133 drops two hard-wired worker ids (14 and 25, the master-class machines of that fleet) from the
    compute-time sample; here the excluded replicas are a parameter (default: the chief, which also checkpoints)."""
    return [x for x in extract_compute_times(fname) if x[1] not in set(exclude_workers)]


def extract_iteration_times(fname: str) -> List[float]:
    out: List[float] = []
    with open(fname) as f:
        for line in f:
            m = re.match(r".*ITERATION TIMES (.*)", line)
            if m:
                out = json.loads(m.group(1))
    return out


def worker_time_stats(compute_times: Sequence[Tuple[float, int, int]]) -> Dict[str, float]:
    """The percentile report of the reference (tools/benchmark.py:60-111)."""
    if not compute_times:
        return {}
    all_times = np.array([t for t, _, _ in compute_times])
    by_iter: Dict[int, List[float]] = {}
    for t, _, it in compute_times:
        by_iter.setdefault(it, []).append(t)
    p95 = [np.percentile(v, 95, method="nearest") for v in by_iter.values()]
    p99 = [np.percentile(v, 99, method="nearest") for v in by_iter.values()]
    p100 = [np.percentile(v, 100, method="nearest") for v in by_iter.values()]
    return {"stdev": float(np.std(all_times)), "max": float(np.max(all_times)), "mean": float(np.mean(all_times)),
            "p80": float(np.percentile(all_times, 80)), "p90": float(np.percentile(all_times, 90)),
            "p95": float(np.percentile(all_times, 95)), "p99": float(np.percentile(all_times, 99)),
            "mean_iter_p95": float(np.mean(p95)), "median_iter_p95": float(np.median(p95)),
            "mean_iter_p99": float(np.mean(p99)), "median_iter_p99": float(np.median(p99)),
            "mean_iter_p100": float(np.mean(p100)), "median_iter_p100": float(np.median(p100))}


def print_worker_sorted_times(fname: str) -> Dict[str, float]:
    print("File: %s\n-----------------------------" % fname)
    st = worker_time_stats(extract_compute_times(fname))
    for k, v in st.items():
        print("%s: %g" % (k, v))
    return st


# ---- figures ----------------------------------------------------------------------------------------------
def _series(outdir: str, pick):
    out = []
    for fname in sorted(glob.glob(os.path.join(outdir, "*evaluator*"))):
        t, l, p, s = extract_times_losses_precision(fname)
        xs, ys = pick(t, l, p, s)
        out.append((os.path.basename(fname).replace("_out_evaluator", ""), xs, ys))
    return out


def plot_time_loss(outdir: str, dest: str = ".") -> str:
    return line_plot(os.path.join(dest, "time_loss.png"), _series(outdir, lambda t, l, p, s: (t, l)),
                     "time (s)", "loss", logy=True)


def plot_time_step(outdir: str, dest: str = ".") -> str:
    return line_plot(os.path.join(dest, "time_step.png"), _series(outdir, lambda t, l, p, s: (t, s)), "time (s)", "step")


def plot_time_precision(outdir: str, dest: str = ".") -> str:
    return line_plot(os.path.join(dest, "time_precision.png"), _series(outdir, lambda t, l, p, s: (t, p)),
                     "time (s)", "precision")


def _device_eval_curve(train_dir: str):
    rows = np.load(os.path.join(train_dir, "worker0_eval.npy")).reshape(-1, 6)
    rows = rows[np.argsort(rows[:, 1], kind="stable")]
    spent = np.concatenate([[0.0], np.cumsum(rows[:-1, 2])])          # evaluation time before each pass began
    t = rows[:, 1] - rows[0, 1] - spent
    acc = rows[:, 4] / np.maximum(rows[:, 3], 1)
    return t.tolist(), acc.tolist()


def plot_device_time_precision(train_dirs, dest: str = ".", labels: Optional[Sequence[str]] = None) -> str:
    """Accuracy against training time from the chief's in-training evaluations (``--eval_every_steps``,
    ``worker0_eval.npy``: global_step, t_begin_unix_s, eval_seconds, examples, correct, mean_loss).  The time axis starts at
    the first evaluation and leaves out the time spent in the evaluations before each point.

    ``train_dirs``: one train dir, or several (e.g. a K sweep, one run per K) drawn as one curve each, named by ``labels``
    (default: the directories' base names)."""
    dirs = [train_dirs] if isinstance(train_dirs, str) else list(train_dirs)
    if labels is None:
        labels = [os.path.basename(os.path.normpath(d)) for d in dirs]
    if len(labels) != len(dirs):
        raise ValueError("%d labels for %d train dirs" % (len(labels), len(dirs)))
    series = [(lab,) + _device_eval_curve(d) for lab, d in zip(labels, dirs)]
    return line_plot(os.path.join(dest, "device_time_precision.png"), series, "training time (s, evaluation excluded)",
                     "precision")


def plot_step_loss(outdir: str, dest: str = ".") -> str:
    return line_plot(os.path.join(dest, "step_losses.png"), _series(outdir, lambda t, l, p, s: (s, l)),
                     "step", "losses", logy=True)


def plot_time_cdfs(outdir: str, dest: str = ".") -> str:
    series = []
    for fname in sorted(glob.glob(os.path.join(outdir, "*master*"))):
        ct = sorted(t for t, _, _ in extract_compute_times(fname))
        if not ct:
            continue
        probs = [(i + 1) / float(len(ct)) for i in range(len(ct))]
        series.append((os.path.basename(fname).replace("_out_master", ""), ct, probs))
        print_worker_sorted_times(fname)
    return line_plot(os.path.join(dest, "time_cdfs.png"), series, "time (s)", "p(x <= x)")


def plot_figs(cfgs: Sequence[Cfg], evaluator_file_name: str = "out_evaluator", outdir: str = "result_dir",
              n_iters: int = 300, rerun: bool = True, dest: str = ".") -> List[str]:
    print([x["name"] for x in cfgs])
    if rerun:
        for cfg in cfgs:
            run_tf_and_download_files(n_iters, cfg, evaluator_file_name=evaluator_file_name, outdir=outdir)
    os.makedirs(dest, exist_ok=True)
    return [plot_time_loss(outdir, dest), plot_time_step(outdir, dest), plot_time_precision(outdir, dest),
            plot_step_loss(outdir, dest), plot_time_cdfs(outdir, dest)]


if __name__ == "__main__":
    print("Usage: python tools/benchmark.py [use_dir dir|select_files cfg1 cfg2...] [--n_iters=N] [--outdir=D]")
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    opts = dict(a[2:].split("=", 1) for a in sys.argv[1:] if a.startswith("--") and "=" in a)
    cfgs: List[Cfg] = []
    if len(args) >= 2 and args[0] == "use_dir":
        cfgs = [load_cfg_from_file(x) for x in sorted(glob.glob(args[1] + "/*"))]
    elif len(args) >= 2 and args[0] == "select_files":
        cfgs = [load_cfg_from_file(x) for x in args[1:]]
    if cfgs:
        plot_figs(cfgs, n_iters=int(opts.get("n_iters", 300)), outdir=opts.get("outdir", "result_dir"),
                  dest=opts.get("dest", "."))
